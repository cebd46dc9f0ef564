package org.apache.spark.sql.b200;

/**
 * JNI face of libsparkb200.so (include/spark_b200.h).  One static native method per C entry point the
 * operators use; handles are jlong, errors surface as B200Exception (non-zero return + sb_last_error()).
 * Compiled only where a JDK exists -- this image has none (see DESIGN.md); the C side is exercised through
 * ctypes with identical signatures, and tests/test_capi_cpu.py checks that every method below has its JNI function.
 */
public final class Native {
  static { System.loadLibrary("sparkb200_jni"); }   // links against libsparkb200.so
  private Native() {}

  // ---- lifecycle, communicator (ExecutorPlugin.init / shutdown) -----------------------------------------------------------
  public static native void init(int deviceOrdinal);
  public static native void shutdown();
  public static native byte[] commGetUniqueId();
  public static native void commInit(int rank, int nranks, byte[] uniqueId);
  public static native long streamCreate();
  public static native void streamDestroy(long stream);
  public static native void streamSynchronize(long stream);
  public static native long hostAlloc(long bytes);      // pinned host memory (sb_host_alloc)
  public static native void hostFree(long address);

  // ---- tables (ColumnarBatch images) --------------------------------------------------------------------------------------
  /** columns: parallel arrays describing Arrow buffers (type, length, nullCount, data / validity BITMAP / offsets addresses). */
  public static native long tableImportHost(int[] types, int[] scales, long[] lengths, long[] nullCounts, long[] data, long[] validity,
                                            long[] offsets, long stream);   // scales: decimals carry precision << 8 | scale, else 0
  public static native long tableNumRows(long table);
  public static native int tableNumColumns(long table);
  public static native long columnNullCount(long table, int column);    // -1 = unknown
  /** D2H of one column into caller-owned native buffers; returns the column's NULL count. */
  public static native long tableExportHost(long table, int column, long data, long validity, long offsets, long stream);
  public static native void tableRetain(long table);
  public static native void tableRelease(long table);
  public static native long tableSelect(long table, int[] columns);
  public static native long tableZip(long a, long b);           // the columns of a then b; equal row counts, shares buffers
  public static native long tableSlice(long table, long begin, long end, long stream);
  public static native long tableConcat(long[] tables, long stream);

  // ---- string keys as order-preserving dictionary codes (the operators do this internally; public for hosts that keep a column
  //      encoded across operators) ---------------------------------------------------------------------------------------------
  /** returns {codes table (one int32 column), dictionary table (one string column, distinct values ascending)} */
  public static native long[] dictionaryEncode(long table, int column, long stream);
  public static native long dictionaryLookup(long table, int column, long dictionary, long stream);
  public static native long dictionaryDecode(long codes, int column, long dictionary, long stream);

  // ---- expressions, FilterExec / ProjectExec --------------------------------------------------------------------------------
  /** postfix sb_expr program built by ExprCompiler; returns a native handle freed with exprFree. */
  public static native long exprCreate(int[] ops, int[] vtypes, int[] args, int[] args2, long[] literals, byte[] bytes, int outType);
  public static native void exprFree(long expr);
  public static native long filterProject(long table, long predicateExpr, long[] projectionExprs, long stream);
  /** string-producing programs (exprCreate with SB_OP_SF_* nodes, outType STRING): one string column each (sb_string_project). */
  public static native long stringProject(long table, long[] programExprs, long stream);

  // ---- ShuffleExchangeExec ------------------------------------------------------------------------------------------------
  /** returns the partitioned table; offsetsOut receives numPartitions + 1 boundaries. */
  public static native long hashPartition(long table, int[] keyCols, int numPartitions, long stream, long[] offsetsOut);
  public static native long roundRobinPartition(long table, int start, int numPartitions, long stream, long[] offsetsOut);
  public static native long rangePartition(long table, int col, boolean ascending, boolean nullsFirst, long bounds, long stream,
                                           long[] offsetsOut);
  public static native long rangeSample(long table, int col, boolean ascending, boolean nullsFirst, long sampleSize, long seed, long stream);
  public static native long rangeDetermineBounds(long sample, boolean ascending, boolean nullsFirst, int numPartitions, long stream);
  public static native long allToAll(long table, long[] partOffsets, int numPartitions, long stream, long[] outPartOffsets);
  public static native long allGather(long table, long stream);
  /** rows of every (rank, partition): [rank * numPartitions + p] (collective) */
  public static native long[] exchangeCounts(long[] partOffsets, int numPartitions, int nranks, long stream);
  /** MapOutputStatistics.bytesByPartitionId summed over the ranks (collective). */
  public static native long[] mapOutputStatistics(long table, long[] partOffsets, int numPartitions, long stream);

  // ---- HashAggregateExec ---------------------------------------------------------------------------------------------------
  public static native long hashAggregate(long table, int mode, int[] keyCols, int[] funcs, long[] inputExprs, long filterExpr,
                                          long expectedGroups, long stream);
  /** aggregation state across the iterator of batches of a partition (TungstenAggregationIterator.processInputs) */
  public static native long aggCreate(int mode, int[] keyCols, int[] funcs, long[] inputExprs, long filterExpr, long expectedGroups);
  public static native void aggUpdate(long state, long table, long stream);
  public static native void aggMerge(long state, long partialTable, long stream);
  public static native long aggFinish(long state, long stream);
  public static native void aggDestroy(long state);

  // ---- SortExec / TakeOrderedAndProjectExec ---------------------------------------------------------------------------------
  public static native long sort(long table, int[] cols, boolean[] ascending, boolean[] nullsFirst, long stream);
  public static native long topN(long table, int[] cols, boolean[] ascending, boolean[] nullsFirst, long k, long stream);

  // ---- joins -----------------------------------------------------------------------------------------------------------------
  public static native long joinBuild(long table, int[] keyCols, long stream);
  public static native long joinProbe(long relation, long probe, int[] keyCols, int joinType, long stream);
  public static native long joinProbeCondition(long relation, long probe, int[] keyCols, int joinType, long conditionExpr, long stream);
  public static native void hashTableRelease(long relation);
  /** the FilterExec below the build side fused into the build (rows failing it never enter the relation); filterExpr 0 = none */
  public static native long joinBuildFiltered(long table, int[] keyCols, long filterExpr, long stream);
  /** FilterExec below the streamed side and ProjectExec above the join fused into the probe; 0 / null = none / all columns */
  public static native long joinProbeFused(long relation, long probe, int[] keyCols, int joinType, long probeFilterExpr,
                                           int[] probeOutCols, int[] buildOutCols, long stream);
  /** joinProbeFused plus runtime filters (InjectRuntimeFilter.scala:47-100: the BloomFilterMightContain FilterExec the optimizer puts on
   *  the application side): streamed column runtimeFilterCols[i] is tested against the prefilter of the single-key relation
   *  runtimeFilterRelations[i] (built from the creation side with joinBuild) inside the candidate pass; INNER / LEFT_SEMI only */
  public static native long joinProbeRuntimeFiltered(long relation, long probe, int[] keyCols, int joinType, long probeFilterExpr,
                                                     int[] probeOutCols, int[] buildOutCols, int[] runtimeFilterCols,
                                                     long[] runtimeFilterRelations, long stream);

  // ---- WindowExec / ExpandExec -------------------------------------------------------------------------------------------------------
  /** one entry per window expression: SB_WIN_* code, input column, frame type (0 rows / 1 range), bounds (Long.MIN_VALUE /
   *  Long.MAX_VALUE = UNBOUNDED, 0 = CURRENT ROW, negative = PRECEDING), parameter (ntile buckets, lag / lead offset) */
  public static native long window(long table, int[] partitionCols, int[] orderCols, boolean[] ascending, boolean[] nullsFirst,
                                   int[] funcs, int[] inputCols, int[] frameTypes, long[] lowers, long[] uppers, long[] params,
                                   long stream);
  /** projectionExprs: nlists * ncols expression handles, list-major */
  public static native long expand(long table, long[] projectionExprs, int nlists, int ncols, long stream);

  // ---- fused exchange: map side + transport in one collective (sb_shuffle_exchange) --------------------------------------------
  public static native long shuffleExchange(long table, int[] keyCols, int numPartitions, long stream, long[] outPartOffsets);

  // ---- columnar scan: Parquet column-chunk pages in pinned host memory -> Arrow columns in HBM ---------------------------------
  /** page table of one column chunk: rows of {encoding, numValues, valuesOffset, valuesBytes, defOffset, defBytes}; the last row is
   *  {dictOffset, dictCount, 0, 0, 0, 0} */
  public static native long[] parquetChunkPages(long chunkAddress, long chunkBytes, int maxDefLevel);
  /** one entry per column: decoded type / scale / Parquet physical type, the chunk's host address and size, and its page table as
   *  parquetChunkPages returned it */
  public static native long scanDecode(int[] types, int[] scales, int[] physicalTypes, long[] chunkAddresses, long[] chunkBytes,
                                       long[][] pageTables, long stream);
  /** spans of the pages of a chunk whose pages may be compressed (codec: parquet.thrift CompressionCodec, UNCOMPRESSED or SNAPPY):
   *  rows of {pageType, encoding, numValues, levelsBytes, bodyOffset, compressedBytes, uncompressedBytes, valuesCompressed,
   *  headerBytes} */
  public static native long[] parquetPageSpans(long chunkAddress, long chunkBytes, int codec, int maxDefLevel);
  /** scanDecode for chunks whose pages may be SNAPPY-compressed: one entry per column, its span table as parquetPageSpans
   *  returned it */
  public static native long scanDecodeCompressed(int[] types, int[] scales, int[] physicalTypes, int[] codecs, int[] maxDefLevels,
                                                 long[] chunkAddresses, long[] chunkBytes, long[][] spanTables, long stream);
}
