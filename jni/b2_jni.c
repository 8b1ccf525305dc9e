/* b2_jni.c — the thin JNI layer between the RAPIDS Accelerator's Java natives and libb200sql.so (north_star: "Scala host
 * code calls, through a thin JNI/C-ABI layer, hand-written sm_90a CUDA kernels").
 *
 * Every function below is the native side of a method the reference's Scala code calls on `ai.rapids.cudf.*` /
 * `com.nvidia.spark.rapids.jni.*` (classes of the un-vendored spark-rapids-jni jar, pom.xml:834-836): it unwraps the `long`
 * handles, calls ONE C-ABI entry point of include/b200sql.h and maps the status code to the Java exception the Scala code
 * already handles (INTEGRATION.md §1).  Method names and parameter lists follow the public cudf-java API the call sites
 * use; the jar's private native signatures are not in /root/reference, so a maintainer adjusts parameter lists where the
 * pinned jar differs (the bodies stay one call each).
 *
 * Build (needs a JDK):      make -C jni JAVA_HOME=/path/to/jdk        -> jni/libb2jni.so  (links ../spark-rapids_b200/lib/libb200sql.so)
 * Syntax check (no JDK):    make -C jni check                          (uses jni/stub/jni.h)
 */
#include <jni.h>
#include <stdlib.h>
#include <string.h>
#include "../include/b200sql.h"

/* ---- status -> exception (INTEGRATION.md §1; RmmRapidsRetryIterator.scala:65-203; Plugin.scala:823-848) ---------------------- */
static void b2_throw(JNIEnv* env, int rc) {
  static const char* cls[] = {NULL,
                              "ai/rapids/cudf/CudfException",                        /* B2_ERR_INVALID        */
                              "ai/rapids/cudf/CudaException",                        /* B2_ERR_CUDA           */
                              "com/nvidia/spark/rapids/jni/GpuRetryOOM",             /* B2_ERR_OOM            */
                              "ai/rapids/cudf/CudfColumnSizeOverflowException",      /* B2_ERR_SIZE_OVERFLOW  */
                              "java/lang/UnsupportedOperationException",             /* B2_ERR_UNSUPPORTED    */
                              "ai/rapids/cudf/CudaFatalException"};                  /* B2_ERR_FATAL          */
  if (rc < 1 || rc > 6) rc = 1;
  jclass c = (*env)->FindClass(env, cls[rc]);
  if (c) (*env)->ThrowNew(env, c, b2_last_error());
}
#define B2_JNI(call, fail) do { int rc_ = (call); if (rc_ != B2_OK) { b2_throw(env, rc_); return fail; } } while (0)

/* cudf-java returns a new table as the array of its column handles (Table(long[] cudfColumns)) */
static jlongArray table_to_column_handles(JNIEnv* env, b2_handle table) {
  int32_t n = 0;
  if (b2_table_num_columns(table, &n) != B2_OK) { b2_throw(env, B2_ERR_INVALID); b2_table_close(table); return NULL; }
  jlongArray out = (*env)->NewLongArray(env, n);
  for (int32_t i = 0; out && i < n; i++) {
    b2_handle c = 0;
    if (b2_table_column(table, i, &c) != B2_OK) { b2_throw(env, B2_ERR_INVALID); break; }
    jlong v = (jlong)c;
    (*env)->SetLongArrayRegion(env, out, i, 1, &v);
  }
  b2_table_close(table);   /* the Java Table owns the column references from here on */
  return out;
}
/* a Java long[] of column-view handles -> a temporary table over them */
static int table_of_columns(JNIEnv* env, jlongArray j_cols, b2_handle* out) {
  jsize n = (*env)->GetArrayLength(env, j_cols);
  jlong* cols = (*env)->GetLongArrayElements(env, j_cols, NULL);
  int rc = b2_table_create((const b2_handle*)cols, n, out);
  (*env)->ReleaseLongArrayElements(env, j_cols, cols, JNI_ABORT);
  return rc;
}

/* ---- runtime: Rmm.initialize / Cuda.DEFAULT_STREAM.sync (GpuDeviceManager.scala:349-445) --------------------------------------- */
JNIEXPORT void JNICALL Java_ai_rapids_cudf_Rmm_initializeInternal(JNIEnv* env, jclass cls, jint allocation_mode, jint log_to, jstring path,
                                                                  jlong pool_size, jint device) {
  (void)cls; (void)allocation_mode; (void)log_to; (void)path;
  B2_JNI(b2_init(device, (size_t)pool_size), );
}
JNIEXPORT void JNICALL Java_ai_rapids_cudf_Cuda_streamSynchronize(JNIEnv* env, jclass cls, jlong stream) {
  (void)cls; (void)stream;   /* per-thread default stream: GpuDeviceManager.scala:364-367 */
  B2_JNI(b2_stream_sync(), );
}

/* ---- ColumnVector / ColumnView refcounts (Arm.scala withResource / closeOnExcept) ---------------------------------------------- */
JNIEXPORT void JNICALL Java_ai_rapids_cudf_ColumnVector_deleteCudfColumn(JNIEnv* env, jclass cls, jlong handle) {
  (void)cls;
  B2_JNI(b2_column_close((b2_handle)handle), );
}
JNIEXPORT jlong JNICALL Java_ai_rapids_cudf_ColumnView_getNativeRowCount(JNIEnv* env, jclass cls, jlong handle) {
  (void)cls;
  b2_column_info ci;
  B2_JNI(b2_column_info_get((b2_handle)handle, &ci), 0);
  return (jlong)ci.size;
}
JNIEXPORT jlong JNICALL Java_ai_rapids_cudf_ColumnView_getNativeNullCount(JNIEnv* env, jclass cls, jlong handle) {
  (void)cls;
  b2_column_info ci;
  B2_JNI(b2_column_info_get((b2_handle)handle, &ci), 0);
  return (jlong)ci.null_count;
}

/* ---- a2: Table.filter(mask) (basicPhysicalOperators.scala:1158-1184) ------------------------------------------------------------ */
JNIEXPORT jlongArray JNICALL Java_ai_rapids_cudf_Table_filter(JNIEnv* env, jclass cls, jlong j_table, jlong j_mask) {
  (void)cls;
  b2_handle out = 0;
  B2_JNI(b2_filter_mask((b2_handle)j_table, (b2_handle)j_mask, &out), NULL);
  return table_to_column_handles(env, out);
}

/* ---- a3-a5: Table.groupByAggregate (GpuAggregateExec.scala:562-585) -------------------------------------------------------------
 * aggs: b2_agg_spec fields flattened by the Java side as 5 ints per aggregate (kind, column, out dtype, out scale, out precision) */
JNIEXPORT jlongArray JNICALL Java_ai_rapids_cudf_Table_groupByAggregate(JNIEnv* env, jclass cls, jlong j_table, jintArray j_keys, jintArray j_aggs) {
  (void)cls;
  jsize nk = (*env)->GetArrayLength(env, j_keys), na5 = (*env)->GetArrayLength(env, j_aggs);
  jint* keys = (*env)->GetIntArrayElements(env, j_keys, NULL);
  jint* aggs = (*env)->GetIntArrayElements(env, j_aggs, NULL);
  b2_handle out = 0;
  int rc = nk ? b2_groupby((b2_handle)j_table, (const int32_t*)keys, nk, (const b2_agg_spec*)aggs, na5 / 5, &out)
              : b2_reduce((b2_handle)j_table, (const b2_agg_spec*)aggs, na5 / 5, &out);
  (*env)->ReleaseIntArrayElements(env, j_keys, keys, JNI_ABORT);
  (*env)->ReleaseIntArrayElements(env, j_aggs, aggs, JNI_ABORT);
  if (rc != B2_OK) { b2_throw(env, rc); return NULL; }
  return table_to_column_handles(env, out);
}

/* ---- a6: JoinPrimitives.hashInnerJoin(left keys, right keys, nullsEqual) (GpuHashJoin.scala:309-409) ---------------------------
 * The Java API passes BOTH key tables on every call, so the reference rebuilds the hash table for every stream batch.  The
 * shim keeps the last build (keyed by the build-side table handle + nullsEqual) and reuses it while the Scala iterator
 * (HashJoinIterator, :1374-1553) streams batches against the same build batch: b2_join_build runs once per build batch. */
static __thread b2_handle t_build_keys = 0, t_build_ht = 0;
static __thread int t_build_nulls_equal = -1;
static int cached_build(b2_handle build_keys, int nulls_equal, b2_handle* ht) {
  if (t_build_ht && t_build_keys == build_keys && t_build_nulls_equal == nulls_equal) { *ht = t_build_ht; return B2_OK; }
  if (t_build_ht) { b2_join_hash_table_close(t_build_ht); b2_table_close(t_build_keys); t_build_ht = 0; t_build_keys = 0; }
  int rc = b2_join_build(build_keys, nulls_equal, ht);
  if (rc != B2_OK) return rc;
  b2_table_incref(build_keys);   /* the cache entry keeps the keys alive: a recycled handle value can never alias it */
  t_build_keys = build_keys; t_build_ht = *ht; t_build_nulls_equal = nulls_equal;
  return B2_OK;
}
static jlongArray probe_to_maps(JNIEnv* env, b2_handle ht, b2_handle probe_keys, int kind) {
  b2_handle lm = 0, rm = 0;
  B2_JNI(b2_join_probe(ht, probe_keys, kind, &lm, &rm), NULL);
  jlong maps[2] = {(jlong)lm, (jlong)rm};
  jlongArray out = (*env)->NewLongArray(env, rm ? 2 : 1);
  if (out) (*env)->SetLongArrayRegion(env, out, 0, rm ? 2 : 1, maps);
  return out;   /* GatherMap column handles: [left] or [left, right] */
}
JNIEXPORT jlongArray JNICALL Java_com_nvidia_spark_rapids_jni_JoinPrimitives_hashInnerJoin(JNIEnv* env, jclass cls, jlong left_keys, jlong right_keys,
                                                                                          jboolean nulls_equal) {
  (void)cls;
  b2_handle ht = 0;   /* the RIGHT table is the build side (JoinImpl.innerHashJoinBuildRight, GpuHashJoin.scala:340) */
  B2_JNI(cached_build((b2_handle)right_keys, nulls_equal ? 1 : 0, &ht), NULL);
  return probe_to_maps(env, ht, (b2_handle)left_keys, B2_JOIN_INNER);
}
JNIEXPORT jlongArray JNICALL Java_ai_rapids_cudf_Table_leftJoinGatherMaps(JNIEnv* env, jclass cls, jlong left_keys, jlong right_keys, jboolean nulls_equal) {
  (void)cls;
  b2_handle ht = 0;
  B2_JNI(cached_build((b2_handle)right_keys, nulls_equal ? 1 : 0, &ht), NULL);
  return probe_to_maps(env, ht, (b2_handle)left_keys, B2_JOIN_LEFT_OUTER);
}
JNIEXPORT jlongArray JNICALL Java_ai_rapids_cudf_Table_leftSemiJoinGatherMap(JNIEnv* env, jclass cls, jlong left_keys, jlong right_keys, jboolean nulls_equal) {
  (void)cls;
  b2_handle ht = 0;
  B2_JNI(cached_build((b2_handle)right_keys, nulls_equal ? 1 : 0, &ht), NULL);
  return probe_to_maps(env, ht, (b2_handle)left_keys, B2_JOIN_LEFT_SEMI);
}
JNIEXPORT jlongArray JNICALL Java_ai_rapids_cudf_Table_leftAntiJoinGatherMap(JNIEnv* env, jclass cls, jlong left_keys, jlong right_keys, jboolean nulls_equal) {
  (void)cls;
  b2_handle ht = 0;
  B2_JNI(cached_build((b2_handle)right_keys, nulls_equal ? 1 : 0, &ht), NULL);
  return probe_to_maps(env, ht, (b2_handle)left_keys, B2_JOIN_LEFT_ANTI);
}

/* ---- a7: Table.gather(map, OutOfBoundsPolicy) (JoinGatherer.scala:585-599) ------------------------------------------------------ */
JNIEXPORT jlongArray JNICALL Java_ai_rapids_cudf_Table_gather(JNIEnv* env, jclass cls, jlong table, jlong map, jboolean nullify_oob) {
  (void)cls;
  b2_handle out = 0;
  B2_JNI(b2_gather((b2_handle)table, (b2_handle)map, nullify_oob ? 1 : 0, &out), NULL);
  return table_to_column_handles(env, out);
}

/* ---- a8: Table.sortOrder / orderBy (SortUtils.scala:212-218, 373-400); args = 3 ints per key (column, ascending, nullsFirst) ---- */
JNIEXPORT jlong JNICALL Java_ai_rapids_cudf_Table_sortOrder(JNIEnv* env, jclass cls, jlong table, jintArray j_args) {
  (void)cls;
  jsize n3 = (*env)->GetArrayLength(env, j_args);
  jint* a = (*env)->GetIntArrayElements(env, j_args, NULL);
  b2_handle out = 0;
  int rc = b2_sort_order((b2_handle)table, (const b2_order_by_arg*)a, n3 / 3, &out);
  (*env)->ReleaseIntArrayElements(env, j_args, a, JNI_ABORT);
  if (rc != B2_OK) { b2_throw(env, rc); return 0; }
  return (jlong)out;
}
JNIEXPORT jlongArray JNICALL Java_ai_rapids_cudf_Table_orderBy(JNIEnv* env, jclass cls, jlong table, jintArray j_args) {
  (void)cls;
  jsize n3 = (*env)->GetArrayLength(env, j_args);
  jint* a = (*env)->GetIntArrayElements(env, j_args, NULL);
  b2_handle out = 0;
  int rc = b2_order_by((b2_handle)table, (const b2_order_by_arg*)a, n3 / 3, &out);
  (*env)->ReleaseIntArrayElements(env, j_args, a, JNI_ABORT);
  if (rc != B2_OK) { b2_throw(env, rc); return NULL; }
  return table_to_column_handles(env, out);
}

/* ---- a8: Table.merge / upperBound / lowerBound, the natives GpuOutOfCoreSortIterator calls through GpuSorter
 * (SortUtils.scala:172-203 upperBound, :249-301 mergeSortAndCloseWithRetry) ----------------------------------------------------- */
JNIEXPORT jlongArray JNICALL Java_ai_rapids_cudf_Table_merge(JNIEnv* env, jclass cls, jlongArray j_tables, jintArray j_args) {
  (void)cls;
  jsize nt = (*env)->GetArrayLength(env, j_tables), n3 = (*env)->GetArrayLength(env, j_args);
  jlong* ts = (*env)->GetLongArrayElements(env, j_tables, NULL);
  jint* a = (*env)->GetIntArrayElements(env, j_args, NULL);
  b2_handle out = 0;
  int rc = b2_merge_sorted((const b2_handle*)ts, nt, (const b2_order_by_arg*)a, n3 / 3, &out);
  (*env)->ReleaseLongArrayElements(env, j_tables, ts, JNI_ABORT);
  (*env)->ReleaseIntArrayElements(env, j_args, a, JNI_ABORT);
  if (rc != B2_OK) { b2_throw(env, rc); return NULL; }
  return table_to_column_handles(env, out);
}
static jlong search_bounds(JNIEnv* env, jlong sorted, jlong values, jintArray j_args, int upper) {
  jsize n3 = (*env)->GetArrayLength(env, j_args);
  jint* a = (*env)->GetIntArrayElements(env, j_args, NULL);
  b2_handle out = 0;
  int rc = b2_search_bounds((b2_handle)sorted, (b2_handle)values, (const b2_order_by_arg*)a, n3 / 3, upper, &out);
  (*env)->ReleaseIntArrayElements(env, j_args, a, JNI_ABORT);
  if (rc != B2_OK) { b2_throw(env, rc); return 0; }
  return (jlong)out;   /* INT32 column of insertion indexes */
}
JNIEXPORT jlong JNICALL Java_ai_rapids_cudf_Table_upperBound(JNIEnv* env, jclass cls, jlong sorted, jlong values, jintArray j_args) {
  (void)cls;
  return search_bounds(env, sorted, values, j_args, 1);
}
JNIEXPORT jlong JNICALL Java_ai_rapids_cudf_Table_lowerBound(JNIEnv* env, jclass cls, jlong sorted, jlong values, jintArray j_args) {
  (void)cls;
  return search_bounds(env, sorted, values, j_args, 0);
}

/* ---- a9: Hash.murmurHash32 (HashFunctions.scala:196-209), Table.partition (GpuHashPartitioningBase.scala:66-80) ------------------ */
JNIEXPORT jlong JNICALL Java_com_nvidia_spark_rapids_jni_Hash_murmurHash32(JNIEnv* env, jclass cls, jint seed, jlongArray j_cols) {
  (void)cls;
  jsize n = (*env)->GetArrayLength(env, j_cols);
  b2_handle table = 0, out = 0;
  int32_t idx[64];
  if (n > 64) { b2_throw(env, B2_ERR_UNSUPPORTED); return 0; }
  for (jsize i = 0; i < n; i++) idx[i] = i;
  B2_JNI(table_of_columns(env, j_cols, &table), 0);
  int rc = b2_murmur3(table, idx, n, seed, &out);
  b2_table_close(table);
  if (rc != B2_OK) { b2_throw(env, rc); return 0; }
  return (jlong)out;
}
JNIEXPORT jlongArray JNICALL Java_ai_rapids_cudf_Table_partition(JNIEnv* env, jclass cls, jlong table, jlong part_ids, jint num_parts, jintArray j_offsets_out) {
  (void)cls;
  b2_handle out = 0;
  int32_t* offs = (int32_t*)malloc(sizeof(int32_t) * (size_t)(num_parts + 1));
  if (!offs) { b2_throw(env, B2_ERR_INVALID); return NULL; }
  int rc = b2_partition_by_ids((b2_handle)table, (b2_handle)part_ids, num_parts, &out, offs);
  if (rc == B2_OK) (*env)->SetIntArrayRegion(env, j_offsets_out, 0, num_parts, (const jint*)offs);   /* cudf returns the partition STARTS */
  free(offs);
  if (rc != B2_OK) { b2_throw(env, rc); return NULL; }
  return table_to_column_handles(env, out);
}

/* ---- a10: Table.readParquet over the HostMemoryBuffer readPartFile built (GpuParquetScan.scala:2089-2127, 3322-3392) ------------ */
JNIEXPORT jlongArray JNICALL Java_ai_rapids_cudf_Table_readParquet(JNIEnv* env, jclass cls, jobjectArray j_names, jlong address, jlong length) {
  (void)cls;
  jsize n = (*env)->GetArrayLength(env, j_names);
  const char* names[256];
  jstring strs[256];
  if (n > 256) { b2_throw(env, B2_ERR_UNSUPPORTED); return NULL; }
  for (jsize i = 0; i < n; i++) {
    strs[i] = (jstring)(*env)->GetObjectArrayElement(env, j_names, i);
    names[i] = (*env)->GetStringUTFChars(env, strs[i], NULL);
  }
  b2_handle out = 0;
  int rc = b2_parquet_decode((const uint8_t*)(intptr_t)address, (int64_t)length, names, n, &out);
  for (jsize i = 0; i < n; i++) { (*env)->ReleaseStringUTFChars(env, strs[i], names[i]); (*env)->DeleteLocalRef(env, strs[i]); }
  if (rc != B2_OK) { b2_throw(env, rc); return NULL; }
  return table_to_column_handles(env, out);
}

/* ---- a12: Table.concatenate (GpuAggregateExec.scala:700-727) -------------------------------------------------------------------- */
JNIEXPORT jlongArray JNICALL Java_ai_rapids_cudf_Table_concatenate(JNIEnv* env, jclass cls, jlongArray j_tables) {
  (void)cls;
  jsize n = (*env)->GetArrayLength(env, j_tables);
  jlong* t = (*env)->GetLongArrayElements(env, j_tables, NULL);
  b2_handle out = 0;
  int rc = b2_concat((const b2_handle*)t, n, &out);
  (*env)->ReleaseLongArrayElements(env, j_tables, t, JNI_ABORT);
  if (rc != B2_OK) { b2_throw(env, rc); return NULL; }
  return table_to_column_handles(env, out);
}

/* ---- f4: RmmSpark hooks the retry framework drives (RmmRapidsRetryIterator.scala) ------------------------------------------------ */
JNIEXPORT jlong JNICALL Java_com_nvidia_spark_rapids_jni_RmmSpark_spillDeviceMemory(JNIEnv* env, jclass cls, jlong want_bytes) {
  (void)cls;
  int64_t freed = 0;
  B2_JNI(b2_spill((int64_t)want_bytes, &freed), 0);
  return (jlong)freed;
}
