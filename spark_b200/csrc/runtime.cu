// runtime.cu -- lifecycle, streams, HBM buffers and tables (ColumnarBatch images) of libsparkb200.so.
//
// Replaces, for this path only: ExecutorPlugin.init/shutdown, the RowToColumnarExec /
// ColumnarToRowExec transitions (SQLX/Columnar.scala:67-214, 503-546) -- which become plain
// host<->HBM copies of Arrow buffers -- and TaskMemoryManager page allocation (here: the CUDA
// stream-ordered memory pool, no spill).
#include <stdarg.h>
#include <stdexcept>
#include "common.cuh"

namespace sb {

static thread_local std::string g_last_error;
void set_last_error(const std::string &m) { g_last_error = m; }

void fail(int code, const char *fmt, ...) {
  char buf[1024];
  va_list ap;
  va_start(ap, fmt);
  vsnprintf(buf, sizeof(buf), fmt, ap);
  va_end(ap);
  throw Error{code, std::string(buf)};
}

Runtime &rt() {
  static Runtime r;
  return r;
}

void require_init() {
  if (!rt().initialized) fail(SB_ERR_NOT_INITIALIZED, "sb_init has not been called (no CUDA device bound)");
}

// streams created through sb_stream_create that are still alive (buffers free themselves in their stream's order)
static std::mutex g_streams_mu;
static std::vector<cudaStream_t> g_live_streams;
static bool stream_alive(cudaStream_t st) {
  if (st == nullptr) return true;
  std::lock_guard<std::mutex> lk(g_streams_mu);
  for (auto s : g_live_streams)
    if (s == st) return true;
  return false;
}

Buffer *buffer_alloc(int64_t bytes, cudaStream_t st) {
  Buffer *b = new Buffer();
  b->bytes = bytes;
  b->st = st;
  if (bytes > 0) {
    cudaError_t e = cudaMallocAsync(&b->ptr, (size_t)bytes, st);
    if (e != cudaSuccess) {
      delete b;
      cudaGetLastError();
      fail(e == cudaErrorMemoryAllocation ? SB_ERR_OOM : SB_ERR_CUDA, "HBM allocation of %lld bytes failed: %s",
           (long long)bytes, cudaGetErrorString(e));
    }
  }
  return b;
}
Buffer *buffer_borrow(const void *p) {
  Buffer *b = new Buffer();
  b->ptr = const_cast<void *>(p);
  b->owned = false;
  return b;
}
void buffer_retain(Buffer *b) {
  if (b) b->refs.fetch_add(1);
}
void buffer_release(Buffer *b) {
  if (!b) return;
  if (b->refs.fetch_sub(1) == 1) {
    if (b->owned && b->ptr) cudaFreeAsync(b->ptr, stream_alive(b->st) ? b->st : (cudaStream_t)0);
    delete b;
  }
}

Column column_alloc(int32_t type, int32_t scale, int64_t n, bool with_validity, cudaStream_t st) {
  Column c;
  c.type = type;
  c.scale = scale;
  c.length = n;
  c.null_count = with_validity ? -1 : 0;
  int w = type_width(type);
  SB_REQUIRE(w > 0, "column_alloc: variable-width type %d needs explicit buffers", type);
  c.data = buffer_alloc((n * w + 15) / 16 * 16 + 16, st);
  if (with_validity) c.validity = buffer_alloc(bitmap_alloc_bytes(n), st);
  return c;
}
Column column_share(const Column &c) {
  Column r = c;
  buffer_retain(r.data);
  buffer_retain(r.validity);
  buffer_retain(r.offsets);
  return r;
}
void column_release(Column &c) {
  buffer_release(c.data);
  buffer_release(c.validity);
  buffer_release(c.offsets);
  c.data = c.validity = c.offsets = nullptr;
}

sb_table *table_new(int64_t nrows) {
  sb_table *t = new sb_table();
  t->nrows = nrows;
  return t;
}
void table_free(sb_table *t) {
  for (auto &c : t->cols) column_release(c);
  delete t;
}

// ---- per-kernel profiling ---------------------------------------------------------------------
struct ProfEntry {
  std::string name;
  cudaEvent_t e0, e1;
};
static std::mutex g_prof_mu;
static bool g_prof_on = false;
static std::vector<ProfEntry> g_prof_pending;
struct ProfTotal {
  std::string name;
  double ms = 0;
  int64_t launches = 0;
};
static std::vector<ProfTotal> g_prof_totals;

KernelTimer::KernelTimer(const char *name_, cudaStream_t st_) : name(name_), st(st_) {
  if (!g_prof_on) return;
  if (cudaEventCreate(&e0) != cudaSuccess || cudaEventCreate(&e1) != cudaSuccess) {
    e0 = e1 = nullptr;
    return;
  }
  cudaEventRecord(e0, st);
}
KernelTimer::~KernelTimer() {
  if (!e0) return;
  cudaEventRecord(e1, st);
  std::lock_guard<std::mutex> lk(g_prof_mu);
  g_prof_pending.push_back({name, e0, e1});
}

static void prof_drain() {
  for (auto &p : g_prof_pending) {
    float ms = 0;
    if (cudaEventSynchronize(p.e1) == cudaSuccess && cudaEventElapsedTime(&ms, p.e0, p.e1) == cudaSuccess) {
      ProfTotal *t = nullptr;
      for (auto &x : g_prof_totals)
        if (x.name == p.name) t = &x;
      if (!t) {
        g_prof_totals.push_back({p.name, 0, 0});
        t = &g_prof_totals.back();
      }
      t->ms += ms;
      t->launches++;
    }
    cudaEventDestroy(p.e0);
    cudaEventDestroy(p.e1);
  }
  g_prof_pending.clear();
}

}  // namespace sb

using namespace sb;

extern "C" int sb_profile_enable(int32_t on) {
  std::lock_guard<std::mutex> lk(g_prof_mu);
  g_prof_on = on != 0;
  return SB_OK;
}
extern "C" int sb_profile_reset(void) {
  std::lock_guard<std::mutex> lk(g_prof_mu);
  prof_drain();
  g_prof_totals.clear();
  return SB_OK;
}
// every timed section since the last reset as "name=ms/launches;..." (truncated to len)
extern "C" int sb_profile_dump(char *buf, int32_t len) {
  std::lock_guard<std::mutex> lk(g_prof_mu);
  prof_drain();
  std::string out;
  for (auto &x : g_prof_totals) {
    char tmp[160];
    snprintf(tmp, sizeof(tmp), "%s=%.6f/%lld;", x.name.c_str(), x.ms, (long long)x.launches);
    out += tmp;
  }
  if (buf && len > 0) snprintf(buf, (size_t)len, "%s", out.c_str());
  return SB_OK;
}
extern "C" int sb_profile_get(const char *kernel_name, double *out_total_ms, int64_t *out_launches) {
  std::lock_guard<std::mutex> lk(g_prof_mu);
  prof_drain();
  *out_total_ms = 0;
  *out_launches = 0;
  for (auto &x : g_prof_totals)
    if (x.name == kernel_name) {
      *out_total_ms = x.ms;
      *out_launches = x.launches;
    }
  return SB_OK;
}

extern "C" {

const char *sb_last_error(void) { return g_last_error.c_str(); }
int32_t sb_abi_version(void) { return SB_ABI_VERSION; }

int sb_init(int32_t device_ordinal) {
  SB_API_BEGIN
  int ndev = 0;
  cudaError_t e = cudaGetDeviceCount(&ndev);
  if (e != cudaSuccess || ndev == 0) {
    cudaGetLastError();
    fail(SB_ERR_CUDA, "no CUDA device visible (%s): libsparkb200 has no CPU fallback",
         e != cudaSuccess ? cudaGetErrorString(e) : "device count 0");
  }
  SB_REQUIRE(device_ordinal >= 0 && device_ordinal < ndev, "device ordinal %d out of range [0,%d)", device_ordinal, ndev);
  SB_CUDA(cudaSetDevice(device_ordinal));
  cudaDeviceProp prop;
  SB_CUDA(cudaGetDeviceProperties(&prop, device_ordinal));
  if (prop.major != 9 || prop.minor != 0)   // sm_90a code runs on compute capability 9.0 alone
    fail(SB_ERR_UNSUPPORTED, "device %s is sm_%d%d; this library is built for sm_90a (H100) only", prop.name, prop.major, prop.minor);
  Runtime &r = rt();
  r.device = device_ordinal;
  r.num_sms = prop.multiProcessorCount;
  r.cc = prop.major * 10 + prop.minor;
  // keep freed HBM in the stream-ordered pool: operators allocate/free per batch
  cudaMemPool_t pool;
  SB_CUDA(cudaDeviceGetDefaultMemPool(&pool, device_ordinal));
  uint64_t thresh = UINT64_MAX;
  SB_CUDA(cudaMemPoolSetAttribute(pool, cudaMemPoolAttrReleaseThreshold, &thresh));
  r.initialized = true;
  SB_API_END
}

int sb_shutdown(void) {
  SB_API_BEGIN
  if (rt().initialized) {
    cudaDeviceSynchronize();
    rt().initialized = false;
  }
  SB_API_END
}

int sb_device_info(int64_t out[4]) {
  SB_API_BEGIN
  require_init();
  size_t fr = 0, tot = 0;
  SB_CUDA(cudaMemGetInfo(&fr, &tot));
  out[0] = rt().num_sms;
  out[1] = (int64_t)tot;
  out[2] = (int64_t)fr;
  out[3] = rt().cc;
  SB_API_END
}

int64_t sb_kernel_launch_count(void) { return rt().launches.load(); }

int sb_host_alloc(int64_t bytes, void **out) {
  SB_API_BEGIN
  require_init();
  SB_CUDA(cudaHostAlloc(out, (size_t)(bytes > 0 ? bytes : 1), cudaHostAllocDefault));
  SB_API_END
}
int sb_host_free(void *p) {
  SB_API_BEGIN
  if (p) SB_CUDA(cudaFreeHost(p));
  SB_API_END
}

int sb_stream_create(sb_stream **out) {
  SB_API_BEGIN
  require_init();
  sb_stream *s = new sb_stream();
  SB_CUDA(cudaStreamCreateWithFlags(&s->stream, cudaStreamNonBlocking));
  SB_CUDA(cudaEventCreate(&s->ev_start));
  SB_CUDA(cudaEventCreate(&s->ev_stop));
  {
    std::lock_guard<std::mutex> lk(g_streams_mu);
    g_live_streams.push_back(s->stream);
  }
  *out = s;
  SB_API_END
}
int sb_stream_destroy(sb_stream *s) {
  SB_API_BEGIN
  if (s) {
    cudaStreamSynchronize(s->stream);
    {
      std::lock_guard<std::mutex> lk(g_streams_mu);
      for (size_t i = 0; i < g_live_streams.size(); i++)
        if (g_live_streams[i] == s->stream) { g_live_streams.erase(g_live_streams.begin() + i); break; }
    }
    cudaEventDestroy(s->ev_start);
    cudaEventDestroy(s->ev_stop);
    cudaStreamDestroy(s->stream);
    delete s;
  }
  SB_API_END
}
int sb_stream_synchronize(sb_stream *s) {
  SB_API_BEGIN
  require_init();
  SB_CUDA(cudaStreamSynchronize(stream_of(s)));
  SB_API_END
}
int sb_stream_record_start(sb_stream *s) {
  SB_API_BEGIN
  SB_REQUIRE(s, "null stream");
  SB_CUDA(cudaEventRecord(s->ev_start, s->stream));
  SB_API_END
}
int sb_stream_record_stop(sb_stream *s) {
  SB_API_BEGIN
  SB_REQUIRE(s, "null stream");
  SB_CUDA(cudaEventRecord(s->ev_stop, s->stream));
  SB_API_END
}
int sb_stream_elapsed_ms(sb_stream *s, float *out_ms) {
  SB_API_BEGIN
  SB_REQUIRE(s, "null stream");
  SB_CUDA(cudaEventSynchronize(s->ev_stop));
  SB_CUDA(cudaEventElapsedTime(out_ms, s->ev_start, s->ev_stop));
  SB_API_END
}

// ---------------------------------------------------------------------------------------------
static void check_cols(const sb_column *cols, int32_t ncols) {
  SB_REQUIRE(ncols >= 0 && (ncols == 0 || cols), "bad column array");
  for (int i = 0; i < ncols; i++) {
    SB_REQUIRE(cols[i].length == cols[0].length, "column %d has %lld rows, column 0 has %lld", i,
               (long long)cols[i].length, (long long)cols[0].length);
    if (cols[i].type == SB_STRING) SB_REQUIRE(cols[i].offsets || cols[i].length == 0, "string column %d without offsets", i);
    else type_width(cols[i].type);
  }
}

int sb_table_import_host(const sb_column *cols, int32_t ncols, sb_stream *s, sb_table **out) {
  SB_API_BEGIN
  require_init();
  check_cols(cols, ncols);
  cudaStream_t st = stream_of(s);
  int64_t n = ncols ? cols[0].length : 0;
  sb_table *t = table_new(n);
  try {
    for (int i = 0; i < ncols; i++) {
      const sb_column &h = cols[i];
      Column c;
      c.type = h.type;
      c.scale = h.scale;
      c.length = n;
      c.null_count = h.validity ? h.null_count : 0;
      if (h.type == SB_STRING) {
        c.offsets = buffer_alloc((n + 1) * 4 + 16, st);
        int32_t last = 0;
        if (n > 0) {
          SB_CUDA(cudaMemcpyAsync(c.offsets->ptr, h.offsets, (size_t)(n + 1) * 4, cudaMemcpyHostToDevice, st));
          last = h.offsets[n];
        } else {
          SB_CUDA(cudaMemsetAsync(c.offsets->ptr, 0, 4, st));
        }
        c.string_bytes = last;
        c.data = buffer_alloc((int64_t)last + 16, st);   // an arena of up to 2^31 - 1 bytes: the padding must not wrap int32
        if (last > 0) SB_CUDA(cudaMemcpyAsync(c.data->ptr, h.data, (size_t)last, cudaMemcpyHostToDevice, st));
      } else {
        int w = type_width(h.type);
        c.data = buffer_alloc((n * w + 15) / 16 * 16 + 16, st);
        if (n > 0) SB_CUDA(cudaMemcpyAsync(c.data->ptr, h.data, (size_t)(n * w), cudaMemcpyHostToDevice, st));
      }
      if (h.validity) {
        c.validity = buffer_alloc(bitmap_alloc_bytes(n), st);
        SB_CUDA(cudaMemsetAsync(c.validity->ptr, 0, (size_t)bitmap_alloc_bytes(n), st));
        if (n > 0) SB_CUDA(cudaMemcpyAsync(c.validity->ptr, h.validity, (size_t)bitmap_bytes(n), cudaMemcpyHostToDevice, st));
      }
      t->cols.push_back(c);
    }
  } catch (...) {
    table_free(t);
    throw;
  }
  *out = t;
  SB_API_END
}

int sb_table_import_device(const sb_column *cols, int32_t ncols, sb_table **out) {
  SB_API_BEGIN
  require_init();
  check_cols(cols, ncols);
  int64_t n = ncols ? cols[0].length : 0;
  sb_table *t = table_new(n);
  for (int i = 0; i < ncols; i++) {
    const sb_column &h = cols[i];
    Column c;
    c.type = h.type;
    c.scale = h.scale;
    c.length = n;
    c.null_count = h.validity ? h.null_count : 0;
    c.data = buffer_borrow(h.data);
    if (h.validity) c.validity = buffer_borrow(h.validity);
    if (h.type == SB_STRING) {
      c.offsets = buffer_borrow(h.offsets);
      int32_t last = 0;
      if (n > 0) SB_CUDA(cudaMemcpy(&last, h.offsets + n, 4, cudaMemcpyDeviceToHost));
      c.string_bytes = last;
    }
    t->cols.push_back(c);
  }
  *out = t;
  SB_API_END
}

int sb_table_num_rows(const sb_table *t, int64_t *out) {
  SB_API_BEGIN
  SB_REQUIRE(t && out, "null argument");
  *out = t->nrows;
  SB_API_END
}
int sb_table_num_columns(const sb_table *t, int32_t *out) {
  SB_API_BEGIN
  SB_REQUIRE(t && out, "null argument");
  *out = (int32_t)t->cols.size();
  SB_API_END
}
int sb_table_column(const sb_table *t, int32_t i, sb_column *out) {
  SB_API_BEGIN
  SB_REQUIRE(t && out && i >= 0 && i < (int)t->cols.size(), "column index %d out of range", i);
  const Column &c = t->cols[i];
  out->type = c.type;
  out->scale = c.scale;
  out->length = c.length;
  out->null_count = c.null_count;
  out->data = c.d();
  out->validity = c.v();
  out->offsets = c.o();
  SB_API_END
}
int sb_table_string_bytes(const sb_table *t, int32_t i, int64_t *out) {
  SB_API_BEGIN
  SB_REQUIRE(t && out && i >= 0 && i < (int)t->cols.size(), "column index %d out of range", i);
  *out = t->cols[i].string_bytes;
  SB_API_END
}

int sb_table_export_host(const sb_table *t, int32_t i, void *data, uint8_t *validity, int32_t *offsets,
                         int64_t *out_null_count, sb_stream *s) {
  SB_API_BEGIN
  require_init();
  SB_REQUIRE(t && i >= 0 && i < (int)t->cols.size(), "column index %d out of range", i);
  const Column &c = t->cols[i];
  cudaStream_t st = stream_of(s);
  int64_t n = c.length;
  if (c.type == SB_STRING) {
    if (offsets) SB_CUDA(cudaMemcpyAsync(offsets, c.o(), (size_t)(n + 1) * 4, cudaMemcpyDeviceToHost, st));
    if (data && c.string_bytes > 0) SB_CUDA(cudaMemcpyAsync(data, c.d(), (size_t)c.string_bytes, cudaMemcpyDeviceToHost, st));
  } else if (data && n > 0) {
    SB_CUDA(cudaMemcpyAsync(data, c.d(), (size_t)(n * type_width(c.type)), cudaMemcpyDeviceToHost, st));
  }
  int64_t nulls = 0;
  if (c.validity) {
    std::vector<uint8_t> tmp;
    uint8_t *dst = validity;
    if (!dst) {
      tmp.resize((size_t)bitmap_bytes(n) + 1);
      dst = tmp.data();
    }
    if (n > 0) SB_CUDA(cudaMemcpyAsync(dst, c.v(), (size_t)bitmap_bytes(n), cudaMemcpyDeviceToHost, st));
    SB_CUDA(cudaStreamSynchronize(st));
    for (int64_t r = 0; r < n; r++) nulls += !((dst[r >> 3] >> (r & 7)) & 1);
  } else {
    if (validity && n > 0) memset(validity, 0xff, (size_t)bitmap_bytes(n));
    SB_CUDA(cudaStreamSynchronize(st));
  }
  if (out_null_count) *out_null_count = nulls;
  SB_API_END
}

int sb_table_retain(sb_table *t) {
  SB_API_BEGIN
  SB_REQUIRE(t, "null table");
  t->refs.fetch_add(1);
  SB_API_END
}
int sb_table_release(sb_table *t) {
  SB_API_BEGIN
  if (t && t->refs.fetch_sub(1) == 1) table_free(t);
  SB_API_END
}

int sb_table_select(const sb_table *t, const int32_t *cols, int32_t ncols, sb_table **out) {
  SB_API_BEGIN
  SB_REQUIRE(t && out, "null argument");
  sb_table *r = table_new(t->nrows);
  for (int i = 0; i < ncols; i++) {
    if (cols[i] < 0 || cols[i] >= (int)t->cols.size()) {
      table_free(r);
      fail(SB_ERR_INVALID, "select: column %d out of range", cols[i]);
    }
    r->cols.push_back(column_share(t->cols[cols[i]]));
  }
  *out = r;
  SB_API_END
}

int sb_table_zip(const sb_table *a, const sb_table *b, sb_table **out) {
  SB_API_BEGIN
  SB_REQUIRE(a && b && out, "null argument");
  SB_REQUIRE(a->nrows == b->nrows || a->cols.empty() || b->cols.empty(), "zip: row counts differ (%lld vs %lld)",
             (long long)a->nrows, (long long)b->nrows);
  sb_table *r = table_new(a->cols.empty() ? b->nrows : a->nrows);
  for (auto &c : a->cols) r->cols.push_back(column_share(c));
  for (auto &c : b->cols) r->cols.push_back(column_share(c));
  *out = r;
  SB_API_END
}

}  // extern "C"
