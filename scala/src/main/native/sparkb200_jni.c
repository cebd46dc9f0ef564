/*
 * sparkb200_jni.c -- mechanical JNI shim between org.apache.spark.sql.b200.Native and libsparkb200.so.
 * Every function: unpack Java arrays, call the sb_* entry point, throw B200Exception on a non-zero code.
 * Build (needs a JDK for jni.h; none in this image):
 *   gcc -shared -fPIC -I$JAVA_HOME/include -I$JAVA_HOME/include/linux -I../../../../include \
 *       sparkb200_jni.c -L../../../../spark_b200 -lsparkb200 -o libsparkb200_jni.so
 */
#include <jni.h>
#include <stdlib.h>
#include <string.h>
#include "spark_b200.h"

static void throw_if(JNIEnv *env, int rc) {
  if (rc == SB_OK) return;
  jclass cls = (*env)->FindClass(env, "org/apache/spark/sql/b200/B200Exception");
  (*env)->ThrowNew(env, cls, sb_last_error());   /* task fails -> Spark's retry policy applies */
}

JNIEXPORT void JNICALL Java_org_apache_spark_sql_b200_Native_init(JNIEnv *env, jclass c, jint dev) {
  throw_if(env, sb_init(dev));
}

JNIEXPORT jlong JNICALL Java_org_apache_spark_sql_b200_Native_streamCreate(JNIEnv *env, jclass c) {
  sb_stream *s = NULL;
  throw_if(env, sb_stream_create(&s));
  return (jlong)(intptr_t)s;
}

JNIEXPORT jlong JNICALL Java_org_apache_spark_sql_b200_Native_tableImportHost(
    JNIEnv *env, jclass c, jintArray types, jintArray scales, jlongArray lengths, jlongArray nulls, jlongArray data, jlongArray validity,
    jlongArray offsets, jlong stream) {
  jsize n = (*env)->GetArrayLength(env, types);
  jint *t = (*env)->GetIntArrayElements(env, types, NULL), *sc = (*env)->GetIntArrayElements(env, scales, NULL);
  jlong *len = (*env)->GetLongArrayElements(env, lengths, NULL), *nc = (*env)->GetLongArrayElements(env, nulls, NULL);
  jlong *d = (*env)->GetLongArrayElements(env, data, NULL), *v = (*env)->GetLongArrayElements(env, validity, NULL);
  jlong *o = (*env)->GetLongArrayElements(env, offsets, NULL);
  sb_column *cols = (sb_column *)calloc((size_t)n, sizeof(sb_column));
  for (jsize i = 0; i < n; i++) {
    cols[i].type = t[i]; cols[i].scale = sc[i]; cols[i].length = len[i]; cols[i].null_count = nc[i];
    cols[i].data = (const void *)(intptr_t)d[i];            /* OffHeapColumnVector / ArrowBuf address */
    cols[i].validity = (const uint8_t *)(intptr_t)v[i];
    cols[i].offsets = (const int32_t *)(intptr_t)o[i];
  }
  sb_table *out = NULL;
  int rc = sb_table_import_host(cols, n, (sb_stream *)(intptr_t)stream, &out);
  free(cols);
  (*env)->ReleaseIntArrayElements(env, types, t, JNI_ABORT);
  (*env)->ReleaseIntArrayElements(env, scales, sc, JNI_ABORT);
  (*env)->ReleaseLongArrayElements(env, lengths, len, JNI_ABORT);
  (*env)->ReleaseLongArrayElements(env, nulls, nc, JNI_ABORT);
  (*env)->ReleaseLongArrayElements(env, data, d, JNI_ABORT);
  (*env)->ReleaseLongArrayElements(env, validity, v, JNI_ABORT);
  (*env)->ReleaseLongArrayElements(env, offsets, o, JNI_ABORT);
  throw_if(env, rc);
  return (jlong)(intptr_t)out;
}

JNIEXPORT void JNICALL Java_org_apache_spark_sql_b200_Native_tableRelease(JNIEnv *env, jclass c, jlong t) {
  throw_if(env, sb_table_release((sb_table *)(intptr_t)t));
}

JNIEXPORT jlong JNICALL Java_org_apache_spark_sql_b200_Native_hashPartition(JNIEnv *env, jclass c, jlong table, jintArray keyCols,
                                                                            jint n, jlong stream, jlongArray offsetsOut) {
  jsize nk = (*env)->GetArrayLength(env, keyCols);
  jint *k = (*env)->GetIntArrayElements(env, keyCols, NULL);
  jlong *offs = (*env)->GetLongArrayElements(env, offsetsOut, NULL);
  sb_table *out = NULL;
  int rc = sb_hash_partition((const sb_table *)(intptr_t)table, (const int32_t *)k, nk, n, (sb_stream *)(intptr_t)stream, &out,
                             (int64_t *)offs);
  (*env)->ReleaseIntArrayElements(env, keyCols, k, JNI_ABORT);
  (*env)->ReleaseLongArrayElements(env, offsetsOut, offs, 0);
  throw_if(env, rc);
  return (jlong)(intptr_t)out;
}

JNIEXPORT jlong JNICALL Java_org_apache_spark_sql_b200_Native_hashAggregate(
    JNIEnv *env, jclass c, jlong table, jint mode, jintArray keyCols, jintArray funcs, jlongArray inputExprs, jlong filterExpr,
    jlong expectedGroups, jlong stream) {
  jsize nk = (*env)->GetArrayLength(env, keyCols), na = (*env)->GetArrayLength(env, funcs);
  jint *k = (*env)->GetIntArrayElements(env, keyCols, NULL), *f = (*env)->GetIntArrayElements(env, funcs, NULL);
  jlong *in = (*env)->GetLongArrayElements(env, inputExprs, NULL);
  sb_agg_spec *specs = (sb_agg_spec *)calloc((size_t)(na ? na : 1), sizeof(sb_agg_spec));
  for (jsize i = 0; i < na; i++) {
    specs[i].func = f[i] & 0xFFFF;    /* funcs[i] = SB_AGG_* | sb_agg_spec.flags << 16 */
    specs[i].flags = f[i] >> 16;
    if (in[i]) specs[i].input = *(const sb_expr *)(intptr_t)in[i];
  }
  sb_agg_plan plan = {mode, nk, (const int32_t *)k, na, 0, specs, (const sb_expr *)(intptr_t)filterExpr, expectedGroups};
  sb_table *out = NULL;
  int rc = sb_hash_aggregate((const sb_table *)(intptr_t)table, &plan, (sb_stream *)(intptr_t)stream, &out);
  free(specs);
  (*env)->ReleaseIntArrayElements(env, keyCols, k, JNI_ABORT);
  (*env)->ReleaseIntArrayElements(env, funcs, f, JNI_ABORT);
  (*env)->ReleaseLongArrayElements(env, inputExprs, in, JNI_ABORT);
  throw_if(env, rc);
  return (jlong)(intptr_t)out;
}

JNIEXPORT jlong JNICALL Java_org_apache_spark_sql_b200_Native_joinBuild(JNIEnv *env, jclass c, jlong table, jintArray keyCols, jlong stream) {
  jsize nk = (*env)->GetArrayLength(env, keyCols);
  jint *k = (*env)->GetIntArrayElements(env, keyCols, NULL);
  sb_hash_table *ht = NULL;
  int rc = sb_join_build((const sb_table *)(intptr_t)table, (const int32_t *)k, nk, (sb_stream *)(intptr_t)stream, &ht);
  (*env)->ReleaseIntArrayElements(env, keyCols, k, JNI_ABORT);
  throw_if(env, rc);
  return (jlong)(intptr_t)ht;
}

JNIEXPORT jlong JNICALL Java_org_apache_spark_sql_b200_Native_joinProbe(JNIEnv *env, jclass c, jlong rel, jlong probe, jintArray keyCols,
                                                                        jint joinType, jlong stream) {
  jsize nk = (*env)->GetArrayLength(env, keyCols);
  jint *k = (*env)->GetIntArrayElements(env, keyCols, NULL);
  sb_table *out = NULL;
  int rc = sb_join_probe((const sb_hash_table *)(intptr_t)rel, (const sb_table *)(intptr_t)probe, (const int32_t *)k, nk, joinType,
                         (sb_stream *)(intptr_t)stream, &out);
  (*env)->ReleaseIntArrayElements(env, keyCols, k, JNI_ABORT);
  throw_if(env, rc);
  return (jlong)(intptr_t)out;
}

/* ---- the rest of Native.java, same pattern: arrays in, one sb_* call, throw_if ------------------------------------------------- */
#define NATIVE(ret, name) JNIEXPORT ret JNICALL Java_org_apache_spark_sql_b200_Native_##name
#define TBL(x) ((sb_table *)(intptr_t)(x))
#define STR(x) ((sb_stream *)(intptr_t)(x))

NATIVE(void, shutdown)(JNIEnv *env, jclass c) { throw_if(env, sb_shutdown()); }

NATIVE(jbyteArray, commGetUniqueId)(JNIEnv *env, jclass c) {
  uint8_t id[SB_UNIQUE_ID_BYTES];
  throw_if(env, sb_comm_get_unique_id(id));
  jbyteArray out = (*env)->NewByteArray(env, SB_UNIQUE_ID_BYTES);
  (*env)->SetByteArrayRegion(env, out, 0, SB_UNIQUE_ID_BYTES, (const jbyte *)id);
  return out;
}

NATIVE(void, commInit)(JNIEnv *env, jclass c, jint rank, jint nranks, jbyteArray uniqueId) {
  uint8_t id[SB_UNIQUE_ID_BYTES];
  (*env)->GetByteArrayRegion(env, uniqueId, 0, SB_UNIQUE_ID_BYTES, (jbyte *)id);
  throw_if(env, sb_comm_init(rank, nranks, id));
}

NATIVE(void, streamDestroy)(JNIEnv *env, jclass c, jlong stream) { throw_if(env, sb_stream_destroy(STR(stream))); }

NATIVE(jlong, tableNumRows)(JNIEnv *env, jclass c, jlong table) {
  int64_t n = 0;
  throw_if(env, sb_table_num_rows(TBL(table), &n));
  return (jlong)n;
}

/* D2H of one result column into buffers the JVM owns (OffHeapColumnVector / ArrowBuf addresses) */
NATIVE(jlong, tableExportHost)(JNIEnv *env, jclass c, jlong table, jint column, jlong data, jlong validity, jlong offsets, jlong stream) {
  int64_t nulls = 0;
  throw_if(env, sb_table_export_host(TBL(table), column, (void *)(intptr_t)data, (uint8_t *)(intptr_t)validity,
                                     (int32_t *)(intptr_t)offsets, &nulls, STR(stream)));
  return (jlong)nulls;
}

NATIVE(jlong, exprCreate)(JNIEnv *env, jclass c, jintArray ops, jintArray vtypes, jintArray args, jintArray args2, jlongArray literals,
                          jbyteArray bytes, jint outType) {
  jsize n = (*env)->GetArrayLength(env, ops);
  jsize nb = (*env)->GetArrayLength(env, bytes);
  jint *o = (*env)->GetIntArrayElements(env, ops, NULL), *v = (*env)->GetIntArrayElements(env, vtypes, NULL);
  jint *a = (*env)->GetIntArrayElements(env, args, NULL), *a2 = (*env)->GetIntArrayElements(env, args2, NULL);
  jlong *l = (*env)->GetLongArrayElements(env, literals, NULL);          /* doubles travel as their bit pattern */
  sb_expr *e = (sb_expr *)calloc(1, sizeof(sb_expr));
  sb_expr_node *nodes = (sb_expr_node *)calloc((size_t)(n ? n : 1), sizeof(sb_expr_node));
  for (jsize i = 0; i < n; i++) {
    nodes[i].op = o[i]; nodes[i].vtype = v[i]; nodes[i].arg = a[i]; nodes[i].arg2 = a2[i]; nodes[i].lit.i = l[i];
  }
  e->nodes = nodes; e->n = n; e->out_type = outType;
  if (nb > 0) {                                                          /* the string literals' pool (SB_OP_STR_* slices) */
    uint8_t *pool = (uint8_t *)malloc((size_t)nb);
    (*env)->GetByteArrayRegion(env, bytes, 0, nb, (jbyte *)pool);
    e->bytes = pool; e->nbytes = nb;
  }
  (*env)->ReleaseIntArrayElements(env, ops, o, JNI_ABORT);
  (*env)->ReleaseIntArrayElements(env, vtypes, v, JNI_ABORT);
  (*env)->ReleaseIntArrayElements(env, args, a, JNI_ABORT);
  (*env)->ReleaseIntArrayElements(env, args2, a2, JNI_ABORT);
  (*env)->ReleaseLongArrayElements(env, literals, l, JNI_ABORT);
  return (jlong)(intptr_t)e;
}

NATIVE(void, exprFree)(JNIEnv *env, jclass c, jlong expr) {
  sb_expr *e = (sb_expr *)(intptr_t)expr;
  if (e) {
    free((void *)e->nodes);
    free((void *)e->bytes);
    free(e);
  }
}

NATIVE(jlong, filterProject)(JNIEnv *env, jclass c, jlong table, jlong predicateExpr, jlongArray projectionExprs, jlong stream) {
  jsize np = (*env)->GetArrayLength(env, projectionExprs);
  jlong *p = (*env)->GetLongArrayElements(env, projectionExprs, NULL);
  sb_expr *proj = (sb_expr *)calloc((size_t)(np ? np : 1), sizeof(sb_expr));
  for (jsize i = 0; i < np; i++) proj[i] = *(const sb_expr *)(intptr_t)p[i];
  sb_table *out = NULL;
  int rc = sb_filter_project(TBL(table), (const sb_expr *)(intptr_t)predicateExpr, proj, np, STR(stream), &out);
  free(proj);
  (*env)->ReleaseLongArrayElements(env, projectionExprs, p, JNI_ABORT);
  throw_if(env, rc);
  return (jlong)(intptr_t)out;
}

NATIVE(jlong, stringProject)(JNIEnv *env, jclass c, jlong table, jlongArray programExprs, jlong stream) {
  jsize np = (*env)->GetArrayLength(env, programExprs);
  jlong *p = (*env)->GetLongArrayElements(env, programExprs, NULL);
  sb_expr *progs = (sb_expr *)calloc((size_t)(np ? np : 1), sizeof(sb_expr));
  for (jsize i = 0; i < np; i++) progs[i] = *(const sb_expr *)(intptr_t)p[i];
  sb_table *out = NULL;
  int rc = sb_string_project(TBL(table), progs, np, STR(stream), &out);
  free(progs);
  (*env)->ReleaseLongArrayElements(env, programExprs, p, JNI_ABORT);
  throw_if(env, rc);
  return (jlong)(intptr_t)out;
}

NATIVE(jlong, roundRobinPartition)(JNIEnv *env, jclass c, jlong table, jint start, jint n, jlong stream, jlongArray offsetsOut) {
  jlong *offs = (*env)->GetLongArrayElements(env, offsetsOut, NULL);
  sb_table *out = NULL;
  int rc = sb_round_robin_partition(TBL(table), start, n, STR(stream), &out, (int64_t *)offs);
  (*env)->ReleaseLongArrayElements(env, offsetsOut, offs, 0);
  throw_if(env, rc);
  return (jlong)(intptr_t)out;
}

static sb_sort_order *make_orders(JNIEnv *env, jintArray cols, jbooleanArray asc, jbooleanArray nullsFirst, jsize *n_out) {
  jsize n = (*env)->GetArrayLength(env, cols);
  jint *cidx = (*env)->GetIntArrayElements(env, cols, NULL);
  jboolean *a = (*env)->GetBooleanArrayElements(env, asc, NULL), *nf = (*env)->GetBooleanArrayElements(env, nullsFirst, NULL);
  sb_sort_order *o = (sb_sort_order *)calloc((size_t)(n ? n : 1), sizeof(sb_sort_order));
  for (jsize i = 0; i < n; i++) {
    o[i].col = cidx[i]; o[i].ascending = a[i] ? 1 : 0; o[i].nulls_first = nf[i] ? 1 : 0;
  }
  (*env)->ReleaseIntArrayElements(env, cols, cidx, JNI_ABORT);
  (*env)->ReleaseBooleanArrayElements(env, asc, a, JNI_ABORT);
  (*env)->ReleaseBooleanArrayElements(env, nullsFirst, nf, JNI_ABORT);
  *n_out = n;
  return o;
}

NATIVE(jlong, sort)(JNIEnv *env, jclass c, jlong table, jintArray cols, jbooleanArray asc, jbooleanArray nullsFirst, jlong stream) {
  jsize n;
  sb_sort_order *o = make_orders(env, cols, asc, nullsFirst, &n);
  sb_table *out = NULL;
  int rc = sb_sort(TBL(table), o, n, STR(stream), &out);
  free(o);
  throw_if(env, rc);
  return (jlong)(intptr_t)out;
}

NATIVE(jlong, topN)(JNIEnv *env, jclass c, jlong table, jintArray cols, jbooleanArray asc, jbooleanArray nullsFirst, jlong k, jlong stream) {
  jsize n;
  sb_sort_order *o = make_orders(env, cols, asc, nullsFirst, &n);
  sb_table *out = NULL;
  int rc = sb_top_n(TBL(table), o, n, k, STR(stream), &out);
  free(o);
  throw_if(env, rc);
  return (jlong)(intptr_t)out;
}

NATIVE(void, hashTableRelease)(JNIEnv *env, jclass c, jlong relation) {
  throw_if(env, sb_hash_table_release((sb_hash_table *)(intptr_t)relation));
}

NATIVE(jlong, allToAll)(JNIEnv *env, jclass c, jlong table, jlongArray partOffsets, jint n, jlong stream, jlongArray outPartOffsets) {
  jlong *in = (*env)->GetLongArrayElements(env, partOffsets, NULL), *po = (*env)->GetLongArrayElements(env, outPartOffsets, NULL);
  sb_table *out = NULL;
  int rc = sb_all_to_all(TBL(table), (const int64_t *)in, n, STR(stream), &out, (int64_t *)po);
  (*env)->ReleaseLongArrayElements(env, partOffsets, in, JNI_ABORT);
  (*env)->ReleaseLongArrayElements(env, outPartOffsets, po, 0);
  throw_if(env, rc);
  return (jlong)(intptr_t)out;
}

NATIVE(jlong, allGather)(JNIEnv *env, jclass c, jlong table, jlong stream) {
  sb_table *out = NULL;
  throw_if(env, sb_all_gather(TBL(table), STR(stream), &out));
  return (jlong)(intptr_t)out;
}


/* ---- round 2 additions ---------------------------------------------------------------------------------------------------------- */
NATIVE(void, streamSynchronize)(JNIEnv *env, jclass c, jlong stream) { throw_if(env, sb_stream_synchronize(STR(stream))); }

NATIVE(jlong, hostAlloc)(JNIEnv *env, jclass c, jlong bytes) {
  void *p = NULL;
  throw_if(env, sb_host_alloc(bytes, &p));
  return (jlong)(intptr_t)p;
}
NATIVE(void, hostFree)(JNIEnv *env, jclass c, jlong address) { throw_if(env, sb_host_free((void *)(intptr_t)address)); }

NATIVE(jint, tableNumColumns)(JNIEnv *env, jclass c, jlong table) {
  int32_t n = 0;
  throw_if(env, sb_table_num_columns(TBL(table), &n));
  return n;
}
NATIVE(jlong, columnNullCount)(JNIEnv *env, jclass c, jlong table, jint column) {
  sb_column d;
  throw_if(env, sb_table_column(TBL(table), column, &d));
  return (jlong)(d.validity ? d.null_count : 0);
}
NATIVE(void, tableRetain)(JNIEnv *env, jclass c, jlong table) { throw_if(env, sb_table_retain(TBL(table))); }

NATIVE(jlong, tableSelect)(JNIEnv *env, jclass c, jlong table, jintArray columns) {
  jsize n = (*env)->GetArrayLength(env, columns);
  jint *k = (*env)->GetIntArrayElements(env, columns, NULL);
  sb_table *out = NULL;
  int rc = sb_table_select(TBL(table), (const int32_t *)k, n, &out);
  (*env)->ReleaseIntArrayElements(env, columns, k, JNI_ABORT);
  throw_if(env, rc);
  return (jlong)(intptr_t)out;
}
NATIVE(jlong, tableZip)(JNIEnv *env, jclass c, jlong a, jlong b) {
  sb_table *out = NULL;
  throw_if(env, sb_table_zip(TBL(a), TBL(b), &out));
  return (jlong)(intptr_t)out;
}
NATIVE(jlong, tableSlice)(JNIEnv *env, jclass c, jlong table, jlong begin, jlong end, jlong stream) {
  sb_table *out = NULL;
  throw_if(env, sb_table_slice(TBL(table), begin, end, STR(stream), &out));
  return (jlong)(intptr_t)out;
}
NATIVE(jlong, tableConcat)(JNIEnv *env, jclass c, jlongArray tables, jlong stream) {
  jsize n = (*env)->GetArrayLength(env, tables);
  jlong *t = (*env)->GetLongArrayElements(env, tables, NULL);
  const sb_table **ptrs = (const sb_table **)calloc((size_t)(n ? n : 1), sizeof(*ptrs));
  for (jsize i = 0; i < n; i++) ptrs[i] = TBL(t[i]);
  sb_table *out = NULL;
  int rc = sb_table_concat(ptrs, n, STR(stream), &out);
  free(ptrs);
  (*env)->ReleaseLongArrayElements(env, tables, t, JNI_ABORT);
  throw_if(env, rc);
  return (jlong)(intptr_t)out;
}

NATIVE(jlongArray, dictionaryEncode)(JNIEnv *env, jclass c, jlong table, jint column, jlong stream) {
  sb_table *codes = NULL, *dict = NULL;
  int rc = sb_dictionary_encode(TBL(table), column, STR(stream), &codes, &dict);
  jlongArray out = (*env)->NewLongArray(env, 2);
  if (rc == SB_OK) {
    const jlong h[2] = {(jlong)(intptr_t)codes, (jlong)(intptr_t)dict};
    (*env)->SetLongArrayRegion(env, out, 0, 2, h);
  }
  throw_if(env, rc);
  return out;
}
NATIVE(jlong, dictionaryLookup)(JNIEnv *env, jclass c, jlong table, jint column, jlong dictionary, jlong stream) {
  sb_table *out = NULL;
  throw_if(env, sb_dictionary_lookup(TBL(table), column, TBL(dictionary), STR(stream), &out));
  return (jlong)(intptr_t)out;
}
NATIVE(jlong, dictionaryDecode)(JNIEnv *env, jclass c, jlong codes, jint column, jlong dictionary, jlong stream) {
  sb_table *out = NULL;
  throw_if(env, sb_dictionary_decode(TBL(codes), column, TBL(dictionary), STR(stream), &out));
  return (jlong)(intptr_t)out;
}

NATIVE(jlong, rangePartition)(JNIEnv *env, jclass c, jlong table, jint col, jboolean asc, jboolean nullsFirst, jlong bounds, jlong stream,
                              jlongArray offsetsOut) {
  sb_sort_order o = {col, asc ? 1 : 0, nullsFirst ? 1 : 0, 0};
  jlong *offs = (*env)->GetLongArrayElements(env, offsetsOut, NULL);
  sb_table *out = NULL;
  int rc = sb_range_partition(TBL(table), &o, TBL(bounds), STR(stream), &out, (int64_t *)offs);
  (*env)->ReleaseLongArrayElements(env, offsetsOut, offs, 0);
  throw_if(env, rc);
  return (jlong)(intptr_t)out;
}
NATIVE(jlong, rangeSample)(JNIEnv *env, jclass c, jlong table, jint col, jboolean asc, jboolean nullsFirst, jlong sampleSize, jlong seed,
                           jlong stream) {
  sb_sort_order o = {col, asc ? 1 : 0, nullsFirst ? 1 : 0, 0};
  sb_table *out = NULL;
  throw_if(env, sb_range_sample(TBL(table), &o, sampleSize, (uint64_t)seed, STR(stream), &out));
  return (jlong)(intptr_t)out;
}
NATIVE(jlong, rangeDetermineBounds)(JNIEnv *env, jclass c, jlong sample, jboolean asc, jboolean nullsFirst, jint numPartitions, jlong stream) {
  sb_sort_order o = {0, asc ? 1 : 0, nullsFirst ? 1 : 0, 0};
  sb_table *out = NULL;
  throw_if(env, sb_range_determine_bounds(TBL(sample), &o, numPartitions, STR(stream), &out));
  return (jlong)(intptr_t)out;
}

NATIVE(jlongArray, mapOutputStatistics)(JNIEnv *env, jclass c, jlong table, jlongArray partOffsets, jint n, jlong stream) {
  jlong *in = (*env)->GetLongArrayElements(env, partOffsets, NULL);
  int64_t *bytes = (int64_t *)calloc((size_t)(n > 0 ? n : 1), sizeof(int64_t));
  int rc = sb_map_output_statistics(TBL(table), (const int64_t *)in, n, STR(stream), bytes);
  (*env)->ReleaseLongArrayElements(env, partOffsets, in, JNI_ABORT);
  jlongArray out = (*env)->NewLongArray(env, n);
  if (rc == SB_OK) (*env)->SetLongArrayRegion(env, out, 0, n, (const jlong *)bytes);
  free(bytes);
  throw_if(env, rc);
  return out;
}

/* aggregation state: the plan is deep-copied by sb_hash_agg_create, so the temporaries die here */
NATIVE(jlong, aggCreate)(JNIEnv *env, jclass c, jint mode, jintArray keyCols, jintArray funcs, jlongArray inputExprs, jlong filterExpr,
                         jlong expectedGroups) {
  jsize nk = (*env)->GetArrayLength(env, keyCols), na = (*env)->GetArrayLength(env, funcs);
  jint *k = (*env)->GetIntArrayElements(env, keyCols, NULL), *f = (*env)->GetIntArrayElements(env, funcs, NULL);
  jlong *in = (*env)->GetLongArrayElements(env, inputExprs, NULL);
  sb_agg_spec *specs = (sb_agg_spec *)calloc((size_t)(na ? na : 1), sizeof(sb_agg_spec));
  for (jsize i = 0; i < na; i++) {
    specs[i].func = f[i] & 0xFFFF;    /* funcs[i] = SB_AGG_* | sb_agg_spec.flags << 16 */
    specs[i].flags = f[i] >> 16;
    if (in[i]) specs[i].input = *(const sb_expr *)(intptr_t)in[i];
  }
  sb_agg_plan plan = {mode, nk, (const int32_t *)k, na, 0, specs, (const sb_expr *)(intptr_t)filterExpr, expectedGroups};
  sb_agg_state *st = NULL;
  int rc = sb_hash_agg_create(&plan, &st);
  free(specs);
  (*env)->ReleaseIntArrayElements(env, keyCols, k, JNI_ABORT);
  (*env)->ReleaseIntArrayElements(env, funcs, f, JNI_ABORT);
  (*env)->ReleaseLongArrayElements(env, inputExprs, in, JNI_ABORT);
  throw_if(env, rc);
  return (jlong)(intptr_t)st;
}
NATIVE(void, aggUpdate)(JNIEnv *env, jclass c, jlong state, jlong table, jlong stream) {
  throw_if(env, sb_hash_agg_update((sb_agg_state *)(intptr_t)state, TBL(table), STR(stream)));
}
NATIVE(void, aggMerge)(JNIEnv *env, jclass c, jlong state, jlong table, jlong stream) {
  throw_if(env, sb_hash_agg_merge((sb_agg_state *)(intptr_t)state, TBL(table), STR(stream)));
}
NATIVE(jlong, aggFinish)(JNIEnv *env, jclass c, jlong state, jlong stream) {
  sb_table *out = NULL;
  throw_if(env, sb_hash_agg_finish((sb_agg_state *)(intptr_t)state, STR(stream), &out));
  return (jlong)(intptr_t)out;
}
NATIVE(void, aggDestroy)(JNIEnv *env, jclass c, jlong state) { throw_if(env, sb_hash_agg_destroy((sb_agg_state *)(intptr_t)state)); }

NATIVE(jlong, joinProbeCondition)(JNIEnv *env, jclass c, jlong rel, jlong probe, jintArray keyCols, jint joinType, jlong cond, jlong stream) {
  jsize nk = (*env)->GetArrayLength(env, keyCols);
  jint *k = (*env)->GetIntArrayElements(env, keyCols, NULL);
  sb_table *out = NULL;
  int rc = sb_join_probe_condition((const sb_hash_table *)(intptr_t)rel, TBL(probe), (const int32_t *)k, nk, joinType,
                                   (const sb_expr *)(intptr_t)cond, STR(stream), &out);
  (*env)->ReleaseIntArrayElements(env, keyCols, k, JNI_ABORT);
  throw_if(env, rc);
  return (jlong)(intptr_t)out;
}

NATIVE(jlong, window)(JNIEnv *env, jclass c, jlong table, jintArray partCols, jintArray orderCols, jbooleanArray asc, jbooleanArray nullsFirst,
                      jintArray funcs, jintArray inputs, jintArray frameTypes, jlongArray lowers, jlongArray uppers, jlongArray params,
                      jlong stream) {
  jsize np = (*env)->GetArrayLength(env, partCols), no = (*env)->GetArrayLength(env, orderCols), ns = (*env)->GetArrayLength(env, funcs);
  jint *pc = (*env)->GetIntArrayElements(env, partCols, NULL), *oc = (*env)->GetIntArrayElements(env, orderCols, NULL);
  jboolean *a = (*env)->GetBooleanArrayElements(env, asc, NULL), *nf = (*env)->GetBooleanArrayElements(env, nullsFirst, NULL);
  jint *fn = (*env)->GetIntArrayElements(env, funcs, NULL), *in = (*env)->GetIntArrayElements(env, inputs, NULL);
  jint *ft = (*env)->GetIntArrayElements(env, frameTypes, NULL);
  jlong *lo = (*env)->GetLongArrayElements(env, lowers, NULL), *hi = (*env)->GetLongArrayElements(env, uppers, NULL);
  jlong *pa = (*env)->GetLongArrayElements(env, params, NULL);
  sb_sort_order *orders = (sb_sort_order *)calloc((size_t)(no ? no : 1), sizeof(sb_sort_order));
  sb_window_spec *specs = (sb_window_spec *)calloc((size_t)(ns ? ns : 1), sizeof(sb_window_spec));
  for (jsize i = 0; i < no; i++) {
    orders[i].col = oc[i];
    orders[i].ascending = a[i] ? 1 : 0;
    orders[i].nulls_first = nf[i] ? 1 : 0;
  }
  for (jsize i = 0; i < ns; i++) {
    specs[i].func = fn[i];
    specs[i].col = in[i];
    specs[i].frame_type = ft[i];
    specs[i].lower = lo[i];
    specs[i].upper = hi[i];
    specs[i].param = pa[i];
  }
  sb_table *out = NULL;
  int rc = sb_window(TBL(table), (const int32_t *)pc, np, orders, no, specs, ns, STR(stream), &out);
  free(specs);
  free(orders);
  (*env)->ReleaseLongArrayElements(env, params, pa, JNI_ABORT);
  (*env)->ReleaseLongArrayElements(env, uppers, hi, JNI_ABORT);
  (*env)->ReleaseLongArrayElements(env, lowers, lo, JNI_ABORT);
  (*env)->ReleaseIntArrayElements(env, frameTypes, ft, JNI_ABORT);
  (*env)->ReleaseIntArrayElements(env, inputs, in, JNI_ABORT);
  (*env)->ReleaseIntArrayElements(env, funcs, fn, JNI_ABORT);
  (*env)->ReleaseBooleanArrayElements(env, nullsFirst, nf, JNI_ABORT);
  (*env)->ReleaseBooleanArrayElements(env, asc, a, JNI_ABORT);
  (*env)->ReleaseIntArrayElements(env, orderCols, oc, JNI_ABORT);
  (*env)->ReleaseIntArrayElements(env, partCols, pc, JNI_ABORT);
  throw_if(env, rc);
  return (jlong)(intptr_t)out;
}
NATIVE(jlong, expand)(JNIEnv *env, jclass c, jlong table, jlongArray exprs, jint nlists, jint ncols, jlong stream) {
  jsize n = (*env)->GetArrayLength(env, exprs);
  jlong *e = (*env)->GetLongArrayElements(env, exprs, NULL);
  sb_expr *progs = (sb_expr *)calloc((size_t)(n ? n : 1), sizeof(sb_expr));
  for (jsize i = 0; i < n; i++) progs[i] = *(const sb_expr *)(intptr_t)e[i];
  sb_table *out = NULL;
  int rc = n == (jsize)nlists * ncols ? sb_expand(TBL(table), progs, nlists, ncols, STR(stream), &out) : SB_ERR_INVALID;
  free(progs);
  (*env)->ReleaseLongArrayElements(env, exprs, e, JNI_ABORT);
  throw_if(env, rc);
  return (jlong)(intptr_t)out;
}

NATIVE(jlong, joinBuildFiltered)(JNIEnv *env, jclass c, jlong table, jintArray keyCols, jlong filter, jlong stream) {
  jsize nk = (*env)->GetArrayLength(env, keyCols);
  jint *k = (*env)->GetIntArrayElements(env, keyCols, NULL);
  sb_hash_table *out = NULL;
  int rc = sb_join_build_filtered(TBL(table), (const int32_t *)k, nk, (const sb_expr *)(intptr_t)filter, STR(stream), &out);
  (*env)->ReleaseIntArrayElements(env, keyCols, k, JNI_ABORT);
  throw_if(env, rc);
  return (jlong)(intptr_t)out;
}
NATIVE(jlong, joinProbeFused)(JNIEnv *env, jclass c, jlong rel, jlong probe, jintArray keyCols, jint joinType, jlong probeFilter,
                              jintArray probeOut, jintArray buildOut, jlong stream) {
  jsize nk = (*env)->GetArrayLength(env, keyCols);
  jint *k = (*env)->GetIntArrayElements(env, keyCols, NULL);
  jint *po = probeOut ? (*env)->GetIntArrayElements(env, probeOut, NULL) : NULL;
  jint *bo = buildOut ? (*env)->GetIntArrayElements(env, buildOut, NULL) : NULL;
  sb_join_options opt;
  memset(&opt, 0, sizeof(opt));
  opt.probe_filter = (const sb_expr *)(intptr_t)probeFilter;
  opt.probe_out_cols = (const int32_t *)po;
  opt.n_probe_out = po ? (*env)->GetArrayLength(env, probeOut) : 0;
  opt.build_out_cols = (const int32_t *)bo;
  opt.n_build_out = bo ? (*env)->GetArrayLength(env, buildOut) : 0;
  sb_table *out = NULL;
  int rc = sb_join_probe_ex((const sb_hash_table *)(intptr_t)rel, TBL(probe), (const int32_t *)k, nk, joinType, &opt, STR(stream), &out);
  if (bo) (*env)->ReleaseIntArrayElements(env, buildOut, bo, JNI_ABORT);
  if (po) (*env)->ReleaseIntArrayElements(env, probeOut, po, JNI_ABORT);
  (*env)->ReleaseIntArrayElements(env, keyCols, k, JNI_ABORT);
  throw_if(env, rc);
  return (jlong)(intptr_t)out;
}

NATIVE(jlong, joinProbeRuntimeFiltered)(JNIEnv *env, jclass c, jlong rel, jlong probe, jintArray keyCols, jint joinType, jlong probeFilter,
                                        jintArray probeOut, jintArray buildOut, jintArray rfCols, jlongArray rfRelations, jlong stream) {
  jsize nk = (*env)->GetArrayLength(env, keyCols);
  jint *k = (*env)->GetIntArrayElements(env, keyCols, NULL);
  jint *po = probeOut ? (*env)->GetIntArrayElements(env, probeOut, NULL) : NULL;
  jint *bo = buildOut ? (*env)->GetIntArrayElements(env, buildOut, NULL) : NULL;
  jsize nrf = rfCols ? (*env)->GetArrayLength(env, rfCols) : 0;
  jint *rc = nrf ? (*env)->GetIntArrayElements(env, rfCols, NULL) : NULL;
  jlong *rr = nrf ? (*env)->GetLongArrayElements(env, rfRelations, NULL) : NULL;
  const sb_hash_table *rels[8];
  sb_join_options opt;
  memset(&opt, 0, sizeof(opt));
  if (nrf > 8) nrf = 8;
  for (jsize i = 0; i < nrf; i++) rels[i] = (const sb_hash_table *)(intptr_t)rr[i];
  opt.probe_filter = (const sb_expr *)(intptr_t)probeFilter;
  opt.probe_out_cols = (const int32_t *)po;
  opt.n_probe_out = po ? (*env)->GetArrayLength(env, probeOut) : 0;
  opt.build_out_cols = (const int32_t *)bo;
  opt.n_build_out = bo ? (*env)->GetArrayLength(env, buildOut) : 0;
  opt.n_runtime_filters = (int32_t)nrf;
  opt.runtime_filter_cols = (const int32_t *)rc;
  opt.runtime_filter_relations = rels;
  sb_table *out = NULL;
  int rcode = sb_join_probe_ex((const sb_hash_table *)(intptr_t)rel, TBL(probe), (const int32_t *)k, nk, joinType, &opt, STR(stream), &out);
  if (rr) (*env)->ReleaseLongArrayElements(env, rfRelations, rr, JNI_ABORT);
  if (rc) (*env)->ReleaseIntArrayElements(env, rfCols, rc, JNI_ABORT);
  if (bo) (*env)->ReleaseIntArrayElements(env, buildOut, bo, JNI_ABORT);
  if (po) (*env)->ReleaseIntArrayElements(env, probeOut, po, JNI_ABORT);
  (*env)->ReleaseIntArrayElements(env, keyCols, k, JNI_ABORT);
  throw_if(env, rcode);
  return (jlong)(intptr_t)out;
}

NATIVE(jlong, shuffleExchange)(JNIEnv *env, jclass c, jlong table, jintArray keyCols, jint n, jlong stream, jlongArray offsetsOut) {
  jsize nk = (*env)->GetArrayLength(env, keyCols);
  jint *k = (*env)->GetIntArrayElements(env, keyCols, NULL);
  jlong *offs = (*env)->GetLongArrayElements(env, offsetsOut, NULL);
  sb_table *out = NULL;
  int rc = sb_shuffle_exchange(TBL(table), (const int32_t *)k, nk, n, STR(stream), &out, (int64_t *)offs);
  (*env)->ReleaseIntArrayElements(env, keyCols, k, JNI_ABORT);
  (*env)->ReleaseLongArrayElements(env, offsetsOut, offs, 0);
  throw_if(env, rc);
  return (jlong)(intptr_t)out;
}

/* page tables travel as long[6 * (npages + 1)]: npages rows of sb_page fields, then {dict_offset, dict_count, 0, 0, 0, 0} */
#define SB_JNI_MAX_PAGES 65536
NATIVE(jlongArray, parquetChunkPages)(JNIEnv *env, jclass c, jlong chunk, jlong nbytes, jint maxDef) {
  sb_page *pages = (sb_page *)calloc(SB_JNI_MAX_PAGES, sizeof(sb_page));
  int32_t npages = 0, dict_count = 0;
  int64_t dict_offset = -1;
  int rc = sb_parquet_chunk_pages((const uint8_t *)(intptr_t)chunk, nbytes, maxDef, pages, SB_JNI_MAX_PAGES, &npages, &dict_offset, &dict_count);
  jlongArray out = NULL;
  if (rc == SB_OK) {
    jlong *flat = (jlong *)calloc((size_t)(npages + 1) * 6, sizeof(jlong));
    for (int32_t i = 0; i < npages; i++) {
      flat[6 * i + 0] = pages[i].encoding;
      flat[6 * i + 1] = pages[i].num_values;
      flat[6 * i + 2] = pages[i].values_offset;
      flat[6 * i + 3] = pages[i].values_bytes;
      flat[6 * i + 4] = pages[i].def_offset;
      flat[6 * i + 5] = pages[i].def_bytes;
    }
    flat[6 * npages + 0] = dict_offset;
    flat[6 * npages + 1] = dict_count;
    out = (*env)->NewLongArray(env, (npages + 1) * 6);
    (*env)->SetLongArrayRegion(env, out, 0, (npages + 1) * 6, flat);
    free(flat);
  }
  free(pages);
  throw_if(env, rc);
  return out;
}
NATIVE(jlong, scanDecode)(JNIEnv *env, jclass c, jintArray types, jintArray scales, jintArray phys, jlongArray addrs, jlongArray sizes,
                          jobjectArray pageTables, jlong stream) {
  jsize ncols = (*env)->GetArrayLength(env, types);
  jint *ty = (*env)->GetIntArrayElements(env, types, NULL), *sc = (*env)->GetIntArrayElements(env, scales, NULL);
  jint *ph = (*env)->GetIntArrayElements(env, phys, NULL);
  jlong *ad = (*env)->GetLongArrayElements(env, addrs, NULL), *sz = (*env)->GetLongArrayElements(env, sizes, NULL);
  sb_column_chunk *chunks = (sb_column_chunk *)calloc((size_t)(ncols ? ncols : 1), sizeof(sb_column_chunk));
  sb_page **owned = (sb_page **)calloc((size_t)(ncols ? ncols : 1), sizeof(sb_page *));
  for (jsize i = 0; i < ncols; i++) {
    jlongArray pt = (jlongArray)(*env)->GetObjectArrayElement(env, pageTables, i);
    jsize words = (*env)->GetArrayLength(env, pt);
    jlong *flat = (*env)->GetLongArrayElements(env, pt, NULL);
    int32_t npages = (int32_t)(words / 6) - 1;
    owned[i] = (sb_page *)calloc((size_t)(npages > 0 ? npages : 1), sizeof(sb_page));
    for (int32_t p = 0; p < npages; p++) {
      owned[i][p].encoding = (int32_t)flat[6 * p + 0];
      owned[i][p].num_values = (int32_t)flat[6 * p + 1];
      owned[i][p].values_offset = flat[6 * p + 2];
      owned[i][p].values_bytes = flat[6 * p + 3];
      owned[i][p].def_offset = flat[6 * p + 4];
      owned[i][p].def_bytes = flat[6 * p + 5];
    }
    chunks[i].type = ty[i];
    chunks[i].scale = sc[i];
    chunks[i].physical_type = ph[i];
    chunks[i].npages = npages;
    chunks[i].data = (const uint8_t *)(intptr_t)ad[i];
    chunks[i].data_bytes = sz[i];
    chunks[i].pages = owned[i];
    chunks[i].dict_offset = flat[6 * npages + 0];
    chunks[i].dict_count = (int32_t)flat[6 * npages + 1];
    chunks[i].value_multiplier = 0;   /* values as stored: the page tables carry no timestamp unit */
    (*env)->ReleaseLongArrayElements(env, pt, flat, JNI_ABORT);
  }
  sb_table *out = NULL;
  int rc = sb_scan_decode(chunks, ncols, STR(stream), &out);
  for (jsize i = 0; i < ncols; i++) free(owned[i]);
  free(owned);
  free(chunks);
  (*env)->ReleaseLongArrayElements(env, sizes, sz, JNI_ABORT);
  (*env)->ReleaseLongArrayElements(env, addrs, ad, JNI_ABORT);
  (*env)->ReleaseIntArrayElements(env, phys, ph, JNI_ABORT);
  (*env)->ReleaseIntArrayElements(env, scales, sc, JNI_ABORT);
  (*env)->ReleaseIntArrayElements(env, types, ty, JNI_ABORT);
  throw_if(env, rc);
  return (jlong)(intptr_t)out;
}

/* span tables travel as long[9 * nspans]: rows of {page_type, encoding, num_values, levels_bytes, body_offset, compressed_bytes,
 * uncompressed_bytes, values_compressed, header_bytes} */
#define SB_JNI_SPAN_WORDS 9
NATIVE(jlongArray, parquetPageSpans)(JNIEnv *env, jclass c, jlong chunk, jlong nbytes, jint codec, jint maxDef) {
  sb_page_span *spans = (sb_page_span *)calloc(SB_JNI_MAX_PAGES, sizeof(sb_page_span));
  int32_t n = 0;
  int rc = sb_parquet_page_spans((const uint8_t *)(intptr_t)chunk, nbytes, codec, maxDef, spans, SB_JNI_MAX_PAGES, &n);
  jlongArray out = NULL;
  if (rc == SB_OK) {
    jlong *flat = (jlong *)calloc((size_t)(n > 0 ? n : 1) * SB_JNI_SPAN_WORDS, sizeof(jlong));
    for (int32_t i = 0; i < n; i++) {
      jlong *w = flat + (size_t)i * SB_JNI_SPAN_WORDS;
      w[0] = spans[i].page_type;
      w[1] = spans[i].encoding;
      w[2] = spans[i].num_values;
      w[3] = spans[i].levels_bytes;
      w[4] = spans[i].body_offset;
      w[5] = spans[i].compressed_bytes;
      w[6] = spans[i].uncompressed_bytes;
      w[7] = spans[i].values_compressed;
      w[8] = spans[i].header_bytes;
    }
    out = (*env)->NewLongArray(env, n * SB_JNI_SPAN_WORDS);
    (*env)->SetLongArrayRegion(env, out, 0, n * SB_JNI_SPAN_WORDS, flat);
    free(flat);
  }
  free(spans);
  throw_if(env, rc);
  return out;
}
NATIVE(jlong, scanDecodeCompressed)(JNIEnv *env, jclass c, jintArray types, jintArray scales, jintArray phys, jintArray codecs, jintArray maxDefs,
                                    jlongArray addrs, jlongArray sizes, jobjectArray spanTables, jlong stream) {
  jsize ncols = (*env)->GetArrayLength(env, types);
  jint *ty = (*env)->GetIntArrayElements(env, types, NULL), *sc = (*env)->GetIntArrayElements(env, scales, NULL);
  jint *ph = (*env)->GetIntArrayElements(env, phys, NULL), *co = (*env)->GetIntArrayElements(env, codecs, NULL);
  jint *md = (*env)->GetIntArrayElements(env, maxDefs, NULL);
  jlong *ad = (*env)->GetLongArrayElements(env, addrs, NULL), *sz = (*env)->GetLongArrayElements(env, sizes, NULL);
  sb_compressed_chunk *chunks = (sb_compressed_chunk *)calloc((size_t)(ncols ? ncols : 1), sizeof(sb_compressed_chunk));
  sb_page_span **owned = (sb_page_span **)calloc((size_t)(ncols ? ncols : 1), sizeof(sb_page_span *));
  for (jsize i = 0; i < ncols; i++) {
    jlongArray st = (jlongArray)(*env)->GetObjectArrayElement(env, spanTables, i);
    jsize words = (*env)->GetArrayLength(env, st);
    jlong *flat = (*env)->GetLongArrayElements(env, st, NULL);
    int32_t n = (int32_t)(words / SB_JNI_SPAN_WORDS);
    owned[i] = (sb_page_span *)calloc((size_t)(n > 0 ? n : 1), sizeof(sb_page_span));
    for (int32_t p = 0; p < n; p++) {
      const jlong *w = flat + (size_t)p * SB_JNI_SPAN_WORDS;
      owned[i][p].page_type = (int32_t)w[0];
      owned[i][p].encoding = (int32_t)w[1];
      owned[i][p].num_values = (int32_t)w[2];
      owned[i][p].levels_bytes = (int32_t)w[3];
      owned[i][p].body_offset = w[4];
      owned[i][p].compressed_bytes = (int32_t)w[5];
      owned[i][p].uncompressed_bytes = (int32_t)w[6];
      owned[i][p].values_compressed = (int32_t)w[7];
      owned[i][p].header_bytes = (int32_t)w[8];
    }
    chunks[i].type = ty[i];
    chunks[i].scale = sc[i];
    chunks[i].physical_type = ph[i];
    chunks[i].codec = co[i];
    chunks[i].max_def_level = md[i];
    chunks[i].npages = n;
    chunks[i].data = (const uint8_t *)(intptr_t)ad[i];
    chunks[i].data_bytes = sz[i];
    chunks[i].spans = owned[i];
    chunks[i].value_multiplier = 0;
    (*env)->ReleaseLongArrayElements(env, st, flat, JNI_ABORT);
  }
  sb_table *out = NULL;
  int rc = sb_scan_decode_compressed(chunks, ncols, STR(stream), &out);
  for (jsize i = 0; i < ncols; i++) free(owned[i]);
  free(owned);
  free(chunks);
  (*env)->ReleaseLongArrayElements(env, sizes, sz, JNI_ABORT);
  (*env)->ReleaseLongArrayElements(env, addrs, ad, JNI_ABORT);
  (*env)->ReleaseIntArrayElements(env, maxDefs, md, JNI_ABORT);
  (*env)->ReleaseIntArrayElements(env, codecs, co, JNI_ABORT);
  (*env)->ReleaseIntArrayElements(env, phys, ph, JNI_ABORT);
  (*env)->ReleaseIntArrayElements(env, scales, sc, JNI_ABORT);
  (*env)->ReleaseIntArrayElements(env, types, ty, JNI_ABORT);
  throw_if(env, rc);
  return (jlong)(intptr_t)out;
}

NATIVE(jlongArray, exchangeCounts)(JNIEnv *env, jclass c, jlongArray partOffsets, jint n, jint nranks, jlong stream) {
  jlong *in = (*env)->GetLongArrayElements(env, partOffsets, NULL);
  const jsize total = (jsize)n * (nranks > 0 ? nranks : 1);
  int64_t *counts = (int64_t *)calloc((size_t)(total > 0 ? total : 1), sizeof(int64_t));
  int rc = sb_exchange_counts((const int64_t *)in, n, STR(stream), counts);
  (*env)->ReleaseLongArrayElements(env, partOffsets, in, JNI_ABORT);
  jlongArray out = (*env)->NewLongArray(env, total);
  if (rc == SB_OK) (*env)->SetLongArrayRegion(env, out, 0, total, (const jlong *)counts);
  free(counts);
  throw_if(env, rc);
  return out;
}
