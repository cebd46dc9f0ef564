/*
 * spark_b200.h -- the C ABI of libsparkb200.so: an H100-native (sm_90a) implementation of
 * Spark SQL's shuffle / sort / hash-aggregate / hash-join physical-execution hot path.
 *
 * The reference (apache/spark) has no FFI on this path (SURVEY.md 8b): the operators are JVM
 * classes.  Each entry point below therefore replaces the *body* of one reference operator's
 * doExecute()/doExecuteColumnar() and is what a Scala `Gpu*Exec extends SparkPlan` calls through
 * the JNI shim (scala/ + INTEGRATION.md); tests and bench.py bind the same symbols with ctypes.
 * Citations are relative to the reference tree:
 *   SQLX = sql/core/src/main/scala/org/apache/spark/sql/execution
 *   CATJ = sql/catalyst/src/main/java/org/apache/spark/sql
 *
 * Conventions
 *  - plain C types only; every call returns 0 (SB_OK) or an SB_ERR_* code, and
 *    sb_last_error() returns the thread-local message (reference behaviour: operators throw,
 *    the task fails, the scheduler retries -- the JNI shim turns non-zero into an exception).
 *  - column buffers use the Arrow layout the reference exposes through ArrowColumnVector
 *    (CATJ/vectorized/ArrowColumnVector.java:42-47): values buffer, validity BITMAP (LSB first,
 *    NULL pointer = no nulls), int32 offsets for strings.  BOOL is one byte per value like
 *    OffHeapColumnVector (sql/core/src/main/java/.../vectorized/OffHeapColumnVector.java:67-76).
 *  - sb_table handles are device-resident (HBM), immutable and reference counted: the creator
 *    owns one reference ("the executor that creates a ColumnarBatch is responsible for closing
 *    it", SQLX/SparkPlan.scala:355-358 -> sb_table_release == ColumnarBatch.close()).
 *  - no CPU fallback and no spill anywhere: an operator either runs on the GPU or fails.
 */
#ifndef SPARK_B200_H
#define SPARK_B200_H

#include <stdint.h>

#ifdef __cplusplus
extern "C" {
#endif

#define SB_ABI_VERSION 1

/* ---- error codes ---------------------------------------------------------------------- */
#define SB_OK 0
#define SB_ERR_CUDA 1        /* CUDA runtime/driver error (message carries cudaGetErrorString) */
#define SB_ERR_INVALID 2     /* bad argument / malformed plan */
#define SB_ERR_OOM 3         /* HBM exhausted: hard error (reference analogue: aggregateOutOfMemoryError,
                                SQLX/aggregate/HashAggregateExec.scala:998-1001) */
#define SB_ERR_NCCL 4
#define SB_ERR_UNSUPPORTED 5 /* type/operator combination not implemented on the GPU path */
#define SB_ERR_NOT_INITIALIZED 6

/* ---- physical column types (widths follow the reference's row->column converters,
 *      SQLX/Columnar.scala:290-326, 444-457) --------------------------------------------- */
#define SB_BOOL 1        /* 1 byte / value */
#define SB_INT8 2
#define SB_INT16 3
#define SB_INT32 4
#define SB_INT64 5
#define SB_FLOAT32 6
#define SB_FLOAT64 7
#define SB_DATE32 8      /* days since epoch, int32 */
#define SB_TIMESTAMP 9   /* microseconds, int64 */
#define SB_DECIMAL64 10  /* precision <= 18: unscaled int64 + scale */
#define SB_STRING 11     /* int32 offsets + byte arena */
#define SB_DECIMAL128 12 /* precision <= 38: unscaled two's-complement int128, little endian (Arrow decimal128) + scale.  A payload /
                            result type (import, export, gather, slice, concat, SUM / AVG buffers and results); not a key type. */
/* decimal columns: sb_column.scale = scale | precision << 8 (precision 0 = not given: the type's maximum, 18 / 38) */
#define SB_DECIMAL_SCALE(x) ((x) & 0xff)
#define SB_DECIMAL_PRECISION(x) (((x) >> 8) & 0xff)
#define SB_DECIMAL_TYPE(precision, scale) (((precision) << 8) | (scale))

/* One column of a batch: the C image of a ColumnVector (CATJ/vectorized/ColumnVector.java:63-366). */
typedef struct sb_column {
  int32_t type;             /* SB_* */
  int32_t scale;            /* decimals: SB_DECIMAL_TYPE(precision, scale); else 0 */
  int64_t length;           /* rows */
  int64_t null_count;       /* -1 = unknown */
  const void *data;         /* values; SB_STRING: byte arena */
  const uint8_t *validity;  /* Arrow bitmap or NULL */
  const int32_t *offsets;   /* SB_STRING only: length+1 entries */
} sb_column;

/* Streams and ordering.  Every operator takes the sb_stream of the calling task thread and is STREAM-ORDERED on it: its kernels,
 * copies and the allocation / release of its temporaries are enqueued there, and tables it returns may be consumed by later
 * calls on the SAME stream without any synchronisation.  Operators that size their result on the host (filter, join, aggregate,
 * partition, exchange) synchronise the stream where they read the size back, not when they return: the kernels that fill the
 * result may still be running.  To hand a TABLE to another stream or thread, call sb_stream_synchronize on the producing stream
 * first.  A HASH TABLE (a broadcast relation is shared by the tasks of an executor) carries an event recorded at the end of its
 * build: sb_join_probe* on any other stream waits for it on the device, the host never does; release it only after the probes
 * that use it have been enqueued on streams that will outlive them.  sb_table_import_host reads the host buffers asynchronously
 * when they are pinned: keep them alive until the stream is synchronised. */
typedef struct sb_table sb_table;             /* ColumnarBatch resident in HBM */
typedef struct sb_stream sb_stream;           /* one per Spark task thread (CUDA stream + scratch) */
typedef struct sb_hash_table sb_hash_table;   /* HashedRelation resident in HBM */

/* ---- lifecycle: ExecutorPlugin.init / shutdown (core/src/main/java/org/apache/spark/api/plugin/
 *      ExecutorPlugin.java); the GPU ordinal comes from TaskContext.resources()("gpu") ------- */
int sb_init(int32_t device_ordinal);
int sb_shutdown(void);
const char *sb_last_error(void);
int32_t sb_abi_version(void);
/* out[0]=SM count, out[1]=HBM bytes total, out[2]=HBM bytes free, out[3]=compute capability*10 */
int sb_device_info(int64_t out[4]);
/* number of kernels this library has launched since sb_init (for bench.py's gpu_launches) */
int64_t sb_kernel_launch_count(void);

/* per-kernel device timing: when enabled, the hot kernels are bracketed by CUDA events on the stream they
 * are launched on; sb_profile_get returns the summed duration and launch count of one kernel by name
 * (e.g. "agg_update", "partition_scatter", "join_probe") -- bench.py's roofline numbers come from here. */
int sb_profile_enable(int32_t on);
int sb_profile_reset(void);
int sb_profile_get(const char *kernel_name, double *out_total_ms, int64_t *out_launches);
int sb_profile_dump(char *buf, int32_t len);   /* "name=total_ms/launches;..." of every timed section since the last reset */

/* library-wide settings (tests and experiments; production needs none):
 *   "agg_rtc"           1 (default) compile plan-specialised aggregate kernels with NVRTC when a plan first meets a large
 *                       input (the GPU analogue of WholeStageCodegenExec + Janino), 0 = always run the generic kernels
 *   "agg_rtc_min_rows"  inputs with fewer rows run the generic kernels (default 2^20)
 *   "agg_tier"          0 auto, 1 dictionary tier only, 2 shared-memory tier only
 *   "agg_verbose", "expr_interpret_only", "regroup_ldst", "exchange_nccl"   0/1
 *   "join_cand"         join candidate pass: 0 = 16 consecutive rows per thread, 1..3 = lane-strided geometries (default 2)
 *   "sort_variant"      onesweep tile geometry 0..5 (default 4 = 384 threads x 12 keys) */
int sb_config_set(const char *key, int64_t value);
int sb_config_get(const char *key, int64_t *out);

/* pinned host buffers for columns that cross PCIe (the JVM side allocates its off-heap column
 * buffers here so H2D/D2H copies are true DMA) */
int sb_host_alloc(int64_t bytes, void **out);
int sb_host_free(void *p);

int sb_stream_create(sb_stream **out);
int sb_stream_destroy(sb_stream *s);
int sb_stream_synchronize(sb_stream *s);
/* device-side timing on the stream the kernels are launched on (bench.py's roofline numbers) */
int sb_stream_record_start(sb_stream *s);
int sb_stream_record_stop(sb_stream *s);
int sb_stream_elapsed_ms(sb_stream *s, float *out_ms);   /* synchronizes on the stop event */

/* ---- tables: RowToColumnarExec / ColumnarToRowExec replacements (SQLX/Columnar.scala:503-546,
 *      67-214) are host<->HBM copies of Arrow buffers ------------------------------------- */
int sb_table_import_host(const sb_column *cols, int32_t ncols, sb_stream *s, sb_table **out);   /* H2D copy */
int sb_table_import_device(const sb_column *cols, int32_t ncols, sb_table **out);              /* borrow device buffers */
int sb_table_num_rows(const sb_table *t, int64_t *out);
int sb_table_num_columns(const sb_table *t, int32_t *out);
int sb_table_column(const sb_table *t, int32_t i, sb_column *out);   /* device pointers; string: data bytes = offsets[length] */
int sb_table_string_bytes(const sb_table *t, int32_t i, int64_t *out);
/* D2H copy of column i into caller buffers (validity/offsets may be NULL when not needed);
 * out_null_count may be NULL */
int sb_table_export_host(const sb_table *t, int32_t i, void *data, uint8_t *validity, int32_t *offsets,
                         int64_t *out_null_count, sb_stream *s);
int sb_table_retain(sb_table *t);
int sb_table_release(sb_table *t);
/* new table made of a subset / reordering of columns (shares buffers; ProjectExec of plain
 * attribute references) */
int sb_table_select(const sb_table *t, const int32_t *cols, int32_t ncols, sb_table **out);
/* concatenates columns of two tables with equal row counts (shares buffers) */
int sb_table_zip(const sb_table *a, const sb_table *b, sb_table **out);
/* rows [begin, end) as a new table (copies) */
int sb_table_slice(const sb_table *t, int64_t begin, int64_t end, sb_stream *s, sb_table **out);
/* concatenation of tables with identical schemas (copies) */
int sb_table_concat(const sb_table *const *tables, int32_t ntables, sb_stream *s, sb_table **out);

/* ---- string keys: order-preserving dictionary codes (csrc/strings.cu).  Grouping, join and sort keys of type SB_STRING are
 *      compared by Spark byte-wise (UTF8String.equals / compareTo -> ByteArray.compareBinary: unsigned bytes, a proper prefix first;
 *      common/unsafe/src/main/java/org/apache/spark/unsafe/types/UTF8String.java).  sb_hash_aggregate, sb_sort / sb_top_n /
 *      sb_sort_permutation and sb_join_build / sb_join_probe* accept such key columns directly and do this internally; the
 *      entry points are public for hosts that want to keep a column encoded across operators.
 *      encode: out_codes = one SB_INT32 column (validity shared with the input: NULL stays NULL) holding each value's rank among
 *              the column's distinct values; out_dictionary = one SB_STRING column, the distinct values in ascending order.
 *      lookup: codes of column `col` in an EXISTING dictionary; a value that is not in it gets -1.
 *      decode: codes -> strings (NULL, negative or >= dictionary size -> NULL). */
int sb_dictionary_encode(const sb_table *t, int32_t col, sb_stream *s, sb_table **out_codes, sb_table **out_dictionary);
int sb_dictionary_lookup(const sb_table *t, int32_t col, const sb_table *dictionary, sb_stream *s, sb_table **out_codes);
int sb_dictionary_decode(const sb_table *codes, int32_t col, const sb_table *dictionary, sb_stream *s, sb_table **out);

/* ---- columnar scan boundary: Parquet column-chunk pages in host memory -> Arrow columns in HBM.  Replaces the CPU decode of
 *      VectorizedParquetRecordReader.nextBatch / VectorizedColumnReader.readBatch / VectorizedRleValuesReader
 *      (sql/core/src/main/java/org/apache/spark/sql/execution/datasources/parquet/) behind FileSourceScanExec.doExecuteColumnar
 *      (SQLX/DataSourceScanExec.scala:735-760): the ENCODED bytes cross PCIe and the GPU decodes them. ------------------------ */
#define SB_ENC_PLAIN 0
#define SB_ENC_RLE_DICTIONARY 1   /* Parquet RLE_DICTIONARY / PLAIN_DICTIONARY data page: [bit width][RLE / bit-packed hybrid runs] */
#define SB_ENC_RLE_BOOLEAN 2      /* BOOLEAN values as [4-byte length][hybrid runs, bit width 1] (data page V2 writers) */
#define SB_ENC_DELTA_BINARY_PACKED 3      /* INT32 / INT64: [header][blocks of zig-zag min delta, bit widths, packed miniblocks] */
#define SB_ENC_DELTA_LENGTH_BYTE_ARRAY 4  /* BYTE_ARRAY: DELTA_BINARY_PACKED lengths, then the concatenated bytes */
#define SB_ENC_DELTA_BYTE_ARRAY 5         /* BYTE_ARRAY: DELTA_BINARY_PACKED prefix lengths, then DELTA_LENGTH_BYTE_ARRAY suffixes */
#define SB_PHYS_BOOLEAN 0         /* Parquet physical types (parquet.thrift Type) */
#define SB_PHYS_INT32 1
#define SB_PHYS_INT64 2
#define SB_PHYS_FLOAT 4
#define SB_PHYS_DOUBLE 5
#define SB_PHYS_BYTE_ARRAY 6      /* decodes to SB_STRING: PLAIN, dictionary, DELTA_LENGTH_BYTE_ARRAY, DELTA_BYTE_ARRAY */

typedef struct sb_page {            /* one data page; offsets are relative to sb_column_chunk.data */
  int32_t encoding;                 /* SB_ENC_* */
  int32_t num_values;               /* rows of the page, NULLs included */
  int64_t values_offset, values_bytes;
  int64_t def_offset, def_bytes;    /* RLE hybrid of the definition levels (bit width 1, no length prefix); def_bytes == 0: none */
} sb_page;

typedef struct sb_column_chunk {
  int32_t type;                     /* SB_* type of the decoded column */
  int32_t scale;
  int32_t physical_type;            /* SB_PHYS_* */
  int32_t npages;
  const uint8_t *data;              /* HOST bytes of the column chunk as they lie in the file (page headers included) */
  int64_t data_bytes;
  const sb_page *pages;
  int64_t dict_offset;              /* PLAIN dictionary values, or -1 */
  int32_t dict_count;
  int32_t value_multiplier;         /* 0 or 1: values as stored.  Else each decoded INT64 value is multiplied by it (wrapping), in
                                       every encoding: 1000 reads a TIMESTAMP(MILLIS) column as SB_TIMESTAMP microseconds, the
                                       conversion of the reference's LongAsMicrosUpdater */
} sb_column_chunk;

/* host only (no device): page descriptors of a column chunk lying in a Parquet file: Thrift compact PageHeader walk (data page
 * V1 / V2, dictionary page); compressed pages -> SB_ERR_UNSUPPORTED.  The DELTA_BINARY_PACKED header in front of a DELTA_* page's
 * values is validated here (block size in [1, 2^20], miniblock count in [1, block size], miniblock size a multiple of 8, total
 * count not above the page's values: else SB_ERR_INVALID); a DELTA_BYTE_ARRAY page whose first prefix length is not 0 (it would
 * continue the previous page's last value, PARQUET-246) -> SB_ERR_UNSUPPORTED. */
int sb_parquet_chunk_pages(const uint8_t *chunk, int64_t nbytes, int32_t max_def_level, sb_page *out_pages, int32_t pages_cap,
                           int32_t *out_npages, int64_t *out_dict_offset, int32_t *out_dict_count);
/* uncompressed pages only (see sb_scan_decode_compressed): one H2D copy per column chunk, then one decode kernel (a block per page). A call with only fixed-width columns does not
 * synchronise the stream.  A call that decodes SB_STRING columns (physical BYTE_ARRAY) synchronises it once, to read back the
 * arena sizes of all of them together; an arena above 2^31 - 1 bytes is SB_ERR_UNSUPPORTED. */
int sb_scan_decode(const sb_column_chunk *chunks, int32_t ncols, sb_stream *s, sb_table **out);

/* Compressed column chunks.  The host walks the page headers (Parquet never compresses them) into spans; the device does
 * everything that needs the page bodies. */
#define SB_CODEC_UNCOMPRESSED 0     /* parquet.thrift CompressionCodec */
#define SB_CODEC_SNAPPY 1           /* a raw Snappy block per page body (no framing), as parquet-mr and parquet-cpp write it */

typedef struct sb_page_span {       /* one page of a chunk as it lies in the file; offsets relative to the chunk */
  int32_t page_type;                /* 0 DATA_PAGE, 2 DICTIONARY_PAGE, 3 DATA_PAGE_V2 */
  int32_t encoding;                 /* SB_ENC_* (dictionary page: SB_ENC_PLAIN) */
  int32_t num_values;
  int32_t levels_bytes;             /* V2: repetition + definition level bytes, stored uncompressed in front of the values */
  int64_t body_offset;              /* first byte after the page header */
  int32_t compressed_bytes, uncompressed_bytes;
  int32_t values_compressed;        /* 0: UNCOMPRESSED chunk, or a V2 page with is_compressed = false */
  int32_t header_bytes;             /* the page header, which starts at body_offset - header_bytes */
} sb_page_span;

typedef struct sb_compressed_chunk {
  int32_t type, scale, physical_type, codec;   /* codec: SB_CODEC_* */
  int32_t max_def_level, npages;
  int32_t value_multiplier;         /* as sb_column_chunk.value_multiplier (0: values as stored) */
  int32_t pad;
  const uint8_t *data;              /* HOST bytes of the chunk as they lie in the file, headers included */
  int64_t data_bytes;
  const sb_page_span *spans;        /* from sb_parquet_page_spans, the dictionary page included */
} sb_compressed_chunk;

/* host only (no device): the spans of every dictionary and data page of a chunk.  Checks that each body lies inside the chunk,
 * that no size or value count is negative, that the level bytes fit the page, that a dictionary page is PLAIN and that there
 * are no repetition levels (sb_parquet_chunk_pages walks the headers with the same checks).  Whether a page is
 * compressed comes from the codec (the footer's), not from its two sizes.  A codec other than SB_CODEC_UNCOMPRESSED or
 * SB_CODEC_SNAPPY (GZIP, LZO, BROTLI, LZ4, ZSTD, LZ4_RAW) -> SB_ERR_UNSUPPORTED. */
int sb_parquet_page_spans(const uint8_t *chunk, int64_t nbytes, int32_t codec, int32_t max_def_level, sb_page_span *out, int32_t cap,
                          int32_t *out_n);
/* sb_scan_decode for chunks whose pages may be compressed (a chunk may mix V1, V2 and dictionary pages).  One H2D copy per chunk,
 * then scan_snappy decompresses every page of the call into one device image per chunk and scan_resolve_pages reads each page's
 * level length and values header from it.  The call synchronises the stream once for those records: a malformed Snappy stream
 * is SB_ERR_INVALID naming the page, and the page checks of sb_parquet_chunk_pages follow with the same messages.  The decode
 * itself is sb_scan_decode's over the images (one more synchronisation when string columns are decoded). */
int sb_scan_decode_compressed(const sb_compressed_chunk *chunks, int32_t ncols, sb_stream *s, sb_table **out);

/* write-side twin (tests, bench.py): one NULL-free fixed-width column -> a column chunk on the device (out_chunk: one SB_INT8
 * column of bytes) + page descriptors on the host.  dictionary: one-column table of the distinct values in ascending order,
 * or NULL for PLAIN pages.  For an SB_FLOAT32 / SB_FLOAT64 column the dictionary holds the distinct BIT PATTERNS as an SB_INT32 /
 * SB_INT64 column in ascending signed order, so that -0.0 and every NaN payload keep an entry of their own and decode to the bits
 * they were written with (a Parquet dictionary need not be in numeric order). */
int sb_scan_encode(const sb_table *t, int32_t col, const sb_table *dictionary, int64_t page_rows, sb_stream *s, sb_table **out_chunk,
                   sb_page *out_pages, int32_t pages_cap, int32_t *out_npages, int64_t *out_dict_offset, int32_t *out_dict_count);

/* ---- expressions: FilterExec / ProjectExec payload (SQLX/basicPhysicalOperators.scala:47, 245),
 *      postfix programs over the input table's columns.  Null-propagating arithmetic and
 *      comparisons, Kleene AND/OR, non-ANSI wrap-around integers, Divide -> NULL on zero,
 *      double comparison with NaN == NaN and NaN largest (SQLOrderingUtil.compareDoubles). ---- */
#define SB_OP_COL 1        /* push column `arg` */
#define SB_OP_LIT_I64 2    /* push literal lit.i */
#define SB_OP_LIT_F64 3    /* push literal lit.d */
#define SB_OP_LIT_NULL 4
#define SB_OP_ADD 10
#define SB_OP_SUB 11
#define SB_OP_MUL 12
#define SB_OP_DIV 13       /* double division */
#define SB_OP_NEG 14
#define SB_OP_EQ 20
#define SB_OP_NE 21
#define SB_OP_LT 22
#define SB_OP_LE 23
#define SB_OP_GT 24
#define SB_OP_GE 25
#define SB_OP_AND 30
#define SB_OP_OR 31
#define SB_OP_NOT 32
#define SB_OP_ISNULL 33
#define SB_OP_ISNOTNULL 34
#define SB_OP_CAST_F64 40
#define SB_OP_CAST_I64 41
#define SB_OP_CAST_I32 42
/* string tests (UTF8_BINARY: unsigned bytes, UTF8String.binaryCompare).  Leaves: the string column is `arg` (never a COL node: a
 * string COL is only valid as a bare one-node reference), the literal is the slice lit.i = offset << 32 | length of sb_expr.bytes.
 * A NULL string gives NULL.  Comparisons have the column on the left ('x' < s is s > 'x'; s <> 'x' is NOT(STR_EQ)). */
#define SB_OP_STR_EQ 50
#define SB_OP_STR_LT 51
#define SB_OP_STR_LE 52
#define SB_OP_STR_GT 53
#define SB_OP_STR_GE 54
#define SB_OP_STR_IN 55            /* slice = uint32 count, then count records [uint32 length][bytes]; arg2 = 1: the list holds NULL
                                      (no match -> NULL instead of FALSE, predicates.scala In / InSet) */
#define SB_OP_STR_STARTS_WITH 56
#define SB_OP_STR_ENDS_WITH 57
#define SB_OP_STR_CONTAINS 58
#define SB_OP_STR_LIKE 59          /* slice = the pattern (UTF-8); arg2 = the escape character (a code point <= 0xFFFF, usually '\\').
                                      `_` matches one code point, `%` any run of them, newlines included */
#define SB_OP_STR_OCTET_LENGTH 60  /* I32: the byte length; the slice is empty */
#define SB_OP_STR_CHAR_LENGTH 61   /* I32: the code points (Length, UTF8String.numChars: one per lead byte, stepping by the width the
                                      lead byte declares, so ill-formed bytes count as Spark counts them); the slice is empty */

/* string-producing programs (sb_string_project, csrc/strfunc.cu): postfix lists of the nodes below, vtype 0, whose value is a
 * string.  Literal slices are lit.i = offset << 32 | length of sb_expr.bytes, as for the string tests.  Semantics are
 * UTF8String's (UTF8_BINARY, non-ANSI); code points are stepped by the width each lead byte declares.  A value is assembled from
 * at most SB_SF_MAX_RANGES byte ranges (a pad counts as one), which validation checks statically. */
#define SB_OP_SF_COL 70            /* push string column `arg` */
#define SB_OP_SF_LIT 71            /* push the literal slice; arg2 = 1: a NULL string */
#define SB_OP_SF_SUBSTRING 72      /* pop s; push substringSQL(s, pos = arg, len = arg2) */
#define SB_OP_SF_CONCAT 73         /* pop `arg` >= 1 strings; push their concatenation, NULL if any is NULL */
#define SB_OP_SF_CONCAT_WS 74      /* pop `arg` >= 1 strings; push them joined by the literal separator, NULL ones skipped */
#define SB_OP_SF_TRIM 75           /* pop s; arg = 0: trim() (ASCII spaces); arg = 1: trim(trimStr), trimStr = the literal */
#define SB_OP_SF_LTRIM 76
#define SB_OP_SF_RTRIM 77
#define SB_OP_SF_LPAD 78           /* pop s; push lpad(s, len = arg, pad = the literal) */
#define SB_OP_SF_RPAD 79
#define SB_SF_MAX_RANGES 16

/* value class of a node's result */
#define SB_VT_BOOL 1
#define SB_VT_I32 2   /* int8/int16/int32/date32 arithmetic wraps at 32 bits */
#define SB_VT_I64 3
#define SB_VT_F64 4

typedef struct sb_expr_node {
  int32_t op;       /* SB_OP_* */
  int32_t vtype;    /* SB_VT_* of the result */
  int32_t arg;      /* SB_OP_COL, SB_OP_STR_*: column index; comparisons: operand class; CAST: source class */
  int32_t arg2;     /* SB_OP_STR_LIKE: escape code point; SB_OP_STR_IN: 1 = the list holds NULL; 0 everywhere else */
  union { int64_t i; double d; } lit;
} sb_expr_node;

typedef struct sb_expr {
  const sb_expr_node *nodes;   /* postfix order */
  int32_t n;
  int32_t out_type;            /* SB_* type of the materialised result column */
  const uint8_t *bytes;        /* host bytes of the literals of SB_OP_STR_* nodes (NULL when there are none) */
  int64_t nbytes;
} sb_expr;

/* FilterExec + ProjectExec in one pass: rows where `predicate` is TRUE survive (NULL drops the row);
 * predicate may be NULL (no filter); each projection becomes one output column. */
int sb_filter_project(const sb_table *in, const sb_expr *predicate, const sb_expr *projections, int32_t nproj,
                      sb_stream *s, sb_table **out);
/* ProjectExec of string-producing functions: one SB_STRING column per program (SB_OP_SF_* nodes, out_type SB_STRING).  Every
 * program is validated before anything is launched.  The call synchronises the stream once, to read back the arena sizes; an
 * arena above 2^31 - 1 bytes is SB_ERR_UNSUPPORTED naming the output. */
int sb_string_project(const sb_table *in, const sb_expr *programs, int32_t nprog, sb_stream *s, sb_table **out);

/* ---- ShuffleExchangeExec, map side (SQLX/exchange/ShuffleExchangeExec.scala:359-619) ---------
 * partition id = pmod(Murmur3Hash(keys, 42), n): bit-exact with HashPartitioning.partitionIdExpression
 * (sql/catalyst/.../plans/physical/partitioning.scala:339-341; Murmur3_x86_32.java:47-150). */
int sb_partition_ids(const sb_table *in, const int32_t *key_cols, int32_t nkeys, int32_t num_partitions,
                     sb_stream *s, int32_t *out_ids_device);
/* rows regrouped partition-contiguously, arrival order kept inside a partition (what the shuffle writers
 * guarantee per map task); out_offsets_host[num_partitions+1] = partition boundaries. */
int sb_hash_partition(const sb_table *in, const int32_t *key_cols, int32_t nkeys, int32_t num_partitions,
                      sb_stream *s, sb_table **out, int64_t *out_offsets_host);
/* RoundRobinPartitioning (ShuffleExchangeExec.scala:428-442): row i -> (start + 1 + i) mod n */
int sb_round_robin_partition(const sb_table *in, int32_t start, int32_t num_partitions, sb_stream *s,
                             sb_table **out, int64_t *out_offsets_host);

/* ---- HashAggregateExec (SQLX/aggregate/HashAggregateExec.scala:50) with the child FilterExec /
 *      ProjectExec fused in.  Buffer algebra: Sum.scala:113-178, Average.scala:80-135,
 *      Count.scala:94-105, Min/Max. ---------------------------------------------------------- */
#define SB_AGG_SUM 1
#define SB_AGG_AVG 2
#define SB_AGG_COUNT 3        /* count(expr): non-null rows */
#define SB_AGG_COUNT_STAR 4
#define SB_AGG_MIN 5
#define SB_AGG_MAX 6
/* central moments (CentralMomentAgg.scala:49-290): the input is read as DOUBLE (integer and float inputs are converted as
 * Cast(_, DoubleType) does; decimal, string, boolean, date and timestamp inputs are SB_ERR_UNSUPPORTED); NULL inputs are skipped */
#define SB_AGG_VAR_POP 7      /* m2 / n; NULL for n == 0 */
#define SB_AGG_VAR_SAMP 8     /* m2 / (n - 1); NULL for n == 0; for n == 1 NULL, or NaN with SB_AGG_FLAG_NAN_ON_DIVIDE_BY_ZERO */
#define SB_AGG_STDDEV_POP 9   /* sqrt(m2 / n) */
#define SB_AGG_STDDEV_SAMP 10 /* sqrt(m2 / (n - 1)), n == 1 as for VAR_SAMP */

/* sb_agg_spec.flags */
#define SB_AGG_FLAG_NAN_ON_DIVIDE_BY_ZERO 1   /* _SAMP of one row gives NaN, not NULL (nullOnDivideByZero = false, i.e.
                                                 spark.sql.legacy.statisticalAggregate); 0 is Spark's default */

#define SB_AGG_MODE_PARTIAL 1   /* input rows -> keys ++ buffers  (AggUtils.scala:131-208) */
#define SB_AGG_MODE_FINAL 2     /* keys ++ buffers -> keys ++ results */
#define SB_AGG_MODE_COMPLETE 3  /* input rows -> keys ++ results */
#define SB_AGG_MODE_PARTIAL_MERGE 4  /* keys ++ buffers -> keys ++ buffers (AggUtils.scala PartialMerge) */

typedef struct sb_agg_spec {
  int32_t func;        /* SB_AGG_* */
  int32_t flags;       /* SB_AGG_FLAG_* (0 for every function but VAR_SAMP / STDDEV_SAMP) */
  sb_expr input;       /* Partial/Complete: value expression (ignored for COUNT_STAR).
                          Final: ignored -- buffers are read positionally after the keys. */
} sb_agg_spec;

typedef struct sb_agg_plan {
  int32_t mode;                /* SB_AGG_MODE_* */
  int32_t nkeys;
  const int32_t *key_cols;     /* grouping columns of the input table (fixed-width types) */
  int32_t naggs;
  int32_t pad;
  const sb_agg_spec *aggs;
  const sb_expr *filter;       /* fused FilterExec predicate or NULL */
  int64_t expected_groups;     /* hint, 0 = unknown (the usual case: the engine finds the right tier by itself); > 0 sizes the
                                  hash table and picks the tier directly (<= 8: dictionary, else shared-memory / HBM table) */
} sb_agg_plan;

/* Output: key columns, then per aggregate either its buffer columns (Partial: sum -> [sum];
 * avg -> [sum f64, count i64]; count -> [count]; min/max -> [value]; var_* / stddev_* -> [n f64, avg f64, m2 f64], Spark's
 * CentralMomentAgg buffer, (0.0, 0.0, 0.0) for a group without non-NULL input) or its result column (f64 for the moments).
 * Final / PartialMerge read the same buffer columns positionally after the keys. */
int sb_hash_aggregate(const sb_table *in, const sb_agg_plan *plan, sb_stream *s, sb_table **out);
/* build check without a device: compiles the run-time specialisation of a plan given as its raw PlanMeta int32 words
 * (sb_agg_plan_meta_words() of them; layout = csrc/agg_kernels.cuh) and returns the compiler's verdict */
int sb_agg_rtc_compile_check(const int32_t *plan_meta_words, int32_t nwords, char *log, int32_t log_len);
int32_t sb_agg_plan_meta_words(void);
/* kernels the calling thread's last aggregate ran: "generic" or "rtc:<plan hash>" (run-time specialised) */
const char *sb_hash_aggregate_last_plan(void);

/* Aggregation state across the iterator of batches of one partition -- the role of the map that
 * TungstenAggregationIterator.processInputs fills row by row (SQLX/aggregate/TungstenAggregationIterator.scala:206-281):
 *   create(plan)            plan->mode says what finish() returns: PARTIAL / PARTIAL_MERGE -> keys ++ buffers,
 *                           COMPLETE / FINAL -> keys ++ results.  The plan is deep-copied.
 *   update(state, batch)    folds one batch in (PARTIAL / COMPLETE: input rows; FINAL / PARTIAL_MERGE: keys ++ buffers at
 *                           the plan's key_cols / positional buffers).  The batch may be released right after the call.
 *   merge(state, partial)   folds in a table that already has the Partial layout (keys first, then buffers), e.g. the
 *                           finish() of another state or the reduce side of an exchange.
 *   finish(state, &out)     one table for everything seen so far; the state stays usable.
 * No input-sized concatenation happens anywhere (HBM holds one batch plus one row per group seen so far). */
typedef struct sb_agg_state sb_agg_state;
int sb_hash_agg_create(const sb_agg_plan *plan, sb_agg_state **out);
int sb_hash_agg_update(sb_agg_state *state, const sb_table *batch, sb_stream *s);
int sb_hash_agg_merge(sb_agg_state *state, const sb_table *partial, sb_stream *s);
int sb_hash_agg_finish(sb_agg_state *state, sb_stream *s, sb_table **out);
int sb_hash_agg_destroy(sb_agg_state *state);

/* ---- SortExec (SQLX/SortExec.scala:39): stable sort of one partition.  Ordering and NULL
 *      placement follow SortPrefix / PrefixComparators / UnsafeInMemorySorter
 *      (SortOrder.scala:128-242, PrefixComparators.java:28-182, UnsafeInMemorySorter.java:241-262,
 *      348-390) and RadixSort.java:178-259 for the single-column radix path. -------------------- */
typedef struct sb_sort_order {
  int32_t col;
  int32_t ascending;     /* 1 = ASC */
  int32_t nulls_first;   /* 1 = NULLS FIRST */
  int32_t pad;
} sb_sort_order;

int sb_sort(const sb_table *in, const sb_sort_order *orders, int32_t norders, sb_stream *s, sb_table **out);
/* the permutation only (int64 row indices, device buffer of in.num_rows entries) */
int sb_sort_permutation(const sb_table *in, const sb_sort_order *orders, int32_t norders, sb_stream *s,
                        int64_t *out_perm_device);
/* TakeOrderedAndProjectExec (SQLX/limit.scala:310-411): first k rows of the sorted input */
int sb_top_n(const sb_table *in, const sb_sort_order *orders, int32_t norders, int64_t k, sb_stream *s,
             sb_table **out);

/* RangePartitioning for a global sort (core/src/main/scala/org/apache/spark/Partitioner.scala:175-320, used by
 * ShuffleExchangeExec.scala:381-401): partition id = number of range bounds the row's key is strictly greater than under
 * the sort order (getPartition :241-260).  `bounds` is a one-column table holding the numPartitions-1 sorted bounds (from
 * sb_range_sample + sb_range_determine_bounds below, or any other source); rows are regrouped
 * partition-contiguously with arrival order kept, like sb_hash_partition.  One sort column, fixed-width type. */
int sb_range_partition(const sb_table *in, const sb_sort_order *order, const sb_table *bounds, sb_stream *s,
                       sb_table **out, int64_t *out_offsets_host);

/* The sampling half of RangePartitioner (Partitioner.scala:203-216 sketch, :357-388 determineBounds).
 *   sb_range_sample            up to sample_size keys of the order's column drawn uniformly without replacement from this input
 *                              partition, with the weight n / sample.length of :229 as a float32 second column.  The reference's
 *                              reservoir is seeded from the RDD id (XORShiftRandom): which rows are drawn is unpinned.
 *   sb_range_determine_bounds  the candidates of ALL input partitions (concatenate / sb_all_gather the samples) -> at most
 *                              num_partitions - 1 bounds, exactly the reference's walk over the cumulative weights.
 * sampleSizePerPartition = ceil(3 * min(samplePointsPerPartitionHint * partitions, 1e6) / inputPartitions) is the caller's
 * (RangePartitioning in spark_b200/execution.py computes it like :208-211). */
int sb_range_sample(const sb_table *in, const sb_sort_order *order, int64_t sample_size, uint64_t seed, sb_stream *s, sb_table **out);
int sb_range_determine_bounds(const sb_table *sample, const sb_sort_order *order, int32_t num_partitions, sb_stream *s, sb_table **out);

/* ---- WindowExec (SQLX/window/WindowExec.scala:90, WindowFunctionFrame.scala) and ExpandExec (SQLX/ExpandExec.scala:36) --------
 *      sb_window: rows sorted by (partition columns ASC NULLS FIRST, orders) -- the child ordering the reference requires and the
 *      order it emits -- followed by one column per window expression.  Ranking functions ignore the frame.  Frames: ROWS with any
 *      bounds (lower / upper are row offsets, negative = PRECEDING, 0 = CURRENT ROW); RANGE with UNBOUNDED / CURRENT ROW bounds (0)
 *      -- the default frames "RANGE UNBOUNDED PRECEDING .. CURRENT ROW" (with ORDER BY: peers included) and the whole
 *      partition -- and with value offsets over one numeric / date ORDER BY column; min / max need lower = SB_UNBOUNDED_PRECEDING.  Result types: row_number / rank / dense_rank / ntile int32,
 *      percent_rank / cume_dist double, count int64, sum int64 (integral input) or double, avg double, the rest the input type. */
#define SB_WIN_ROW_NUMBER 1
#define SB_WIN_RANK 2
#define SB_WIN_DENSE_RANK 3
#define SB_WIN_PERCENT_RANK 4
#define SB_WIN_CUME_DIST 5
#define SB_WIN_NTILE 6          /* param = buckets */
#define SB_WIN_LAG 7            /* param = offset; NULL outside the partition */
#define SB_WIN_LEAD 8
#define SB_WIN_SUM 9
#define SB_WIN_COUNT 10
#define SB_WIN_AVG 11
#define SB_WIN_MIN 12
#define SB_WIN_MAX 13
#define SB_WIN_FIRST_VALUE 14   /* respect nulls */
#define SB_WIN_LAST_VALUE 15
#define SB_FRAME_ROWS 0
#define SB_FRAME_RANGE 1       /* bounds: UNBOUNDED, 0 = CURRENT ROW (peers included), or int64 VALUE offsets (negative = PRECEDING) over
                                  the single integral / date ORDER BY column */
#define SB_FRAME_RANGE_F64 2   /* the same over a float / double ORDER BY column: offsets are the bits of doubles */
#define SB_UNBOUNDED_PRECEDING INT64_MIN
#define SB_UNBOUNDED_FOLLOWING INT64_MAX
typedef struct sb_window_spec {
  int32_t func;         /* SB_WIN_* */
  int32_t col;          /* input column (ignored by the ranking functions) */
  int32_t frame_type;   /* SB_FRAME_* */
  int32_t pad;
  int64_t lower, upper;
  int64_t param;
} sb_window_spec;
int sb_window(const sb_table *in, const int32_t *partition_cols, int32_t npart, const sb_sort_order *orders, int32_t norders,
              const sb_window_spec *specs, int32_t nspecs, sb_stream *s, sb_table **out);
/* ExpandExec: nlists projection lists of ncols expressions each (projections[l * ncols + c]); every input row yields nlists output
 * rows, list 0 first (the reference's iteration order).  Column c must have one type in every list (NULL literals carry theirs). */
int sb_expand(const sb_table *in, const sb_expr *projections, int32_t nlists, int32_t ncols, sb_stream *s, sb_table **out);

/* ---- joins: BroadcastHashJoinExec / ShuffledHashJoinExec / SortMergeJoinExec replacement
 *      (SQLX/joins/HashJoin.scala:184-400, HashedRelation.scala:136-168).  A row with any NULL key
 *      never matches.  Output = probe(streamed) columns ++ build columns; semi/anti = probe only. ---- */
#define SB_JOIN_INNER 0
#define SB_JOIN_LEFT_OUTER 1   /* streamed side preserved */
#define SB_JOIN_LEFT_SEMI 2
#define SB_JOIN_LEFT_ANTI 3
#define SB_JOIN_FULL_OUTER 4              /* both sides preserved: pairs, streamed rows without a partner, then build rows without one
                                             (ShuffledHashJoinExec.buildSideOrFullOuterJoin, SQLX/joins/ShuffledHashJoinExec.scala:130-330) */
#define SB_JOIN_BUILD_OUTER 5             /* build side preserved (a RIGHT OUTER join whose right side is hashed): pairs + unmatched build rows */
#define SB_JOIN_EXISTENCE 6               /* every streamed row ++ one BOOL column "exists" (HashJoin.existenceJoin, HashJoin.scala:301) */
#define SB_JOIN_LEFT_ANTI_NULL_AWARE 7    /* NOT IN: BroadcastHashJoinExec.scala:137-162 (single key) */

int sb_join_build(const sb_table *build, const int32_t *key_cols, int32_t nkeys, sb_stream *s, sb_hash_table **out);
/* the FilterExec below the build side fused into the build: rows for which `filter` is not TRUE stay out of the relation and
 * the filtered table is never materialised (payload is gathered from `build` by row id at probe time) */
int sb_join_build_filtered(const sb_table *build, const int32_t *key_cols, int32_t nkeys, const sb_expr *filter, sb_stream *s,
                           sb_hash_table **out);
/* what whole-stage codegen fuses around a join on the CPU path (the FilterExec below the streamed side, the ProjectExec above
 * the join), as options of the probe: nothing between scan and join output is materialised */
typedef struct sb_join_options {
  const sb_expr *probe_filter;     /* over the streamed table: rows for which it is not TRUE are not part of the input; or NULL */
  const sb_expr *condition;        /* residual condition over streamed ++ build columns (HashJoin.boundCondition); or NULL */
  const int32_t *probe_out_cols;   /* streamed columns that reach the output (NULL: all) */
  int32_t n_probe_out;
  int32_t n_build_out;
  const int32_t *build_out_cols;   /* build columns that reach the output (NULL: all) */
  /* Runtime filters -- the reference's InjectRuntimeFilter (sql/catalyst/.../optimizer/InjectRuntimeFilter.scala:47-100) plans a
   * BloomFilterMightContain FilterExec on the application side of a join, built from the creation side's join key.  Here the creation
   * side is a single-key relation (sb_join_build*) and its prefilter (exact bitmap or Bloom) is tested on streamed column
   * runtime_filter_cols[i] of the rows that survive the join's own candidate pass (short inputs: of every row): streamed rows whose
   * value cannot be a key of the relation (or is NULL) are not part of the input.  INNER / LEFT_SEMI only; like the reference's filter it may let non-members through, so it is only
   * planned where a later inner join on that column drops them anyway. */
  int32_t n_runtime_filters;
  const int32_t *runtime_filter_cols;
  const sb_hash_table *const *runtime_filter_relations;
} sb_join_options;
int sb_join_probe_ex(const sb_hash_table *ht, const sb_table *probe, const int32_t *key_cols, int32_t nkeys, int32_t join_type,
                     const sb_join_options *options, sb_stream *s, sb_table **out);
int sb_join_probe(const sb_hash_table *ht, const sb_table *probe, const int32_t *key_cols, int32_t nkeys,
                  int32_t join_type, sb_stream *s, sb_table **out);
/* the same with a residual condition over the joined row (streamed columns ++ build columns): HashJoin.scala:144-172
 * boundCondition -- only key matches for which it is TRUE are matches, for every join type */
int sb_join_probe_condition(const sb_hash_table *ht, const sb_table *probe, const int32_t *key_cols, int32_t nkeys,
                            int32_t join_type, const sb_expr *condition, sb_stream *s, sb_table **out);
int sb_hash_table_release(sb_hash_table *ht);

/* ---- synthetic TPC-H-shaped columns (include/sb_synth.h defines the dataset; SURVEY.md 8d: the reference ships no data
 *      generator, BASELINE.json configs[3] asks for on-device generation from a counter-based RNG).  Rows
 *      [first_row, first_row + nrows) of `columns` of table SB_SYNTH_* for a database of n_orders orders. ---- */
int sb_synth_table(int32_t table, const int32_t *columns, int32_t ncols, int64_t n_orders, int64_t first_row,
                   int64_t nrows, uint64_t seed, sb_stream *s, sb_table **out);

/* ---- multi-GPU: one executor process per GPU; the exchange is an NCCL all-to-all over NVLink
 *      instead of shuffle files + Netty fetch (core/.../shuffle/sort/SortShuffleManager.scala:70,
 *      core/.../storage/ShuffleBlockFetcherIterator.scala). ------------------------------------ */
#define SB_UNIQUE_ID_BYTES 128
int sb_comm_get_unique_id(uint8_t out_id[SB_UNIQUE_ID_BYTES]);                 /* rank 0 (driver plugin) */
int sb_comm_init(int32_t rank, int32_t nranks, const uint8_t id[SB_UNIQUE_ID_BYTES]);
int sb_comm_destroy(void);
int sb_comm_rank(int32_t *rank, int32_t *nranks);
/* Ownership of reducer partitions: rank r owns the contiguous range [ceil(r*n/R), ceil((r+1)*n/R))
 * (ShuffledRowRDD maps reducer partitions to tasks; which executor runs which task is the scheduler's choice).
 * Host-only planner used by sb_all_to_all: fills the rows this rank sends to every destination.  No GPU needed. */
int sb_exchange_plan(const int64_t *part_offsets, int32_t num_partitions, int32_t nranks,
                     int64_t *out_send_rows /* nranks */);
/* ShuffleExchangeExec, both sides: `in` is partition-contiguous (from sb_hash_partition) with
 * part_offsets_host; every rank receives the partitions it owns from all ranks.  The result is
 * partition-contiguous (what AQEShuffleReadExec slices by partition offsets); inside a partition the rows
 * are ordered by source rank, arrival order inside a source (fetch order is unspecified in the reference);
 * out_part_offsets_host[num_partitions+1] = partition boundaries of the result (only owned partitions are
 * non-empty).  String columns travel as dictionary codes (csrc/comm.cu).  Collective: all ranks call it in
 * the same order. */
int sb_all_to_all(const sb_table *in, const int64_t *part_offsets_host, int32_t num_partitions, sb_stream *s,
                  sb_table **out, int64_t *out_part_offsets_host);
/* ---- adaptive execution: the statistics of an exchange and the coalescing they drive --------------------------------------------
 * sb_map_output_statistics  MapOutputStatistics.bytesByPartitionId (ShuffleExchangeExec.scala:235-262): bytes every reducer
 *                           partition holds, summed over all map sides (ranks).  Collective when a communicator is up.
 * sb_coalesce_partitions    ShufflePartitionsUtil.coalescePartitions without skew specs (SQLX/adaptive/ShufflePartitionsUtil.scala:
 *                           45-126, 263-369), host only: CoalescedPartitionSpec(start, end) ranges + their data size per shuffle
 *                           (out_data_size[shuffle * nspecs + spec]); *out_nspecs == 0 means "leave the layout as it is". */
/* rows of every (rank, partition): out_counts[rank * num_partitions + p]; collective (one all-gather); no communicator: this rank's */
int sb_exchange_counts(const int64_t *part_offsets_host, int32_t num_partitions, sb_stream *s, int64_t *out_counts);
int sb_map_output_statistics(const sb_table *partitioned, const int64_t *part_offsets_host, int32_t num_partitions, sb_stream *s,
                             int64_t *out_bytes_by_partition);
int sb_coalesce_partitions(const int64_t *const *bytes_by_partition, int32_t nshuffles, int32_t num_partitions,
                           int64_t advisory_target_size, int32_t min_num_partitions, int64_t min_partition_size,
                           int32_t max_reducer_partitions_per_task, int32_t *out_start, int32_t *out_end, int64_t *out_data_size,
                           int32_t *out_nspecs);
/* ShuffleExchangeExec(HashPartitioning) with map side and transport FUSED: one stable multisplit over the destination ranks whose
 * runs are stored straight into the owners' receive windows (remote stores over NVLink -- the scatter kernel is the transport;
 * no local partition-contiguous copy, no push, no copy-out), then one local multisplit into the owned partitions.  The result
 * is partition-contiguous over the owned partitions (rows of a partition: by source rank, arrival order inside a source).
 * Collective.  Same answer as sb_hash_partition + sb_all_to_all up to the order of the source blocks. */
int sb_shuffle_exchange(const sb_table *in, const int32_t *key_cols, int32_t nkeys, int32_t num_partitions, sb_stream *s,
                        sb_table **out, int64_t *out_part_offsets_host);
/* BroadcastExchangeExec (SQLX/exchange/BroadcastExchangeExec.scala:45-279): every rank gets the
 * concatenation of all ranks' tables, in rank order. */
int sb_all_gather(const sb_table *in, sb_stream *s, sb_table **out);

#ifdef __cplusplus
}
#endif
#endif /* SPARK_B200_H */
