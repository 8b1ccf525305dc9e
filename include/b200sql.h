/*
 * b200sql.h — C ABI of libb200sql.so, the H100-native (sm_90a) columnar SQL backend.
 *
 * This is the drop-in boundary (SURVEY.md §8b): the flat C surface that a JNI shim named like
 * the `ai.rapids.cudf.*` / `com.nvidia.spark.rapids.jni.*` natives binds to, so that the RAPIDS
 * Accelerator's unchanged GpuExec operators reach these kernels.  Every entry point cites the
 * reference call site (relative to /root/reference/sql-plugin/src/main/scala/) it stands behind.
 *
 * Conventions (mirroring the cudf-Java handle convention the reference relies on,
 * com/nvidia/spark/rapids/Arm.scala + SURVEY §8b "Handle/ownership"):
 *   - every object is an opaque int64 handle (the "long nativeHandle" of cudf-Java), reference
 *     counted: *_incref / *_close.  Inputs are never consumed; outputs are new objects owned by
 *     the caller.
 *   - every function returns a b2_status; b2_last_error() gives a thread-local message.
 *     B2_ERR_OOM maps to GpuRetryOOM / GpuSplitAndRetryOOM (RmmRapidsRetryIterator.scala:65-203),
 *     B2_ERR_SIZE_OVERFLOW to CudfColumnSizeOverflowException, B2_ERR_FATAL to CudaFatalException
 *     (Plugin.scala:823-848).
 *   - all work is stream ordered on a per-thread stream (GpuDeviceManager.scala:364-367 assumes
 *     the per-thread default stream); b2_stream_sync() is the Cuda.DEFAULT_STREAM.sync() the
 *     reference issues before handing buffers to other threads (GpuPartitioning.scala:93).
 *   - column layout is Arrow/cudf: values buffer, optional 1-bit/row validity (LSB first, padded
 *     to 64 B — GpuBatchUtils.scala:33-41), strings = int32 offsets[n+1] + chars.
 *     DECIMAL128 = 16-byte little-endian two's complement.  Decimal scale here is the SPARK scale
 *     (digits right of the point), i.e. minus the cudf scale (DecimalUtil.scala:24-40).
 */
#ifndef B200SQL_H
#define B200SQL_H

#include <stddef.h>
#include <stdint.h>

#ifdef __cplusplus
extern "C" {
#endif
#if defined(__GNUC__)
#pragma GCC visibility push(default)
#endif

typedef int64_t b2_handle;

typedef enum {
  B2_OK = 0,
  B2_ERR_INVALID = 1,       /* CudfException (logic / bad argument)                      */
  B2_ERR_CUDA = 2,          /* CudaException (recoverable CUDA error)                    */
  B2_ERR_OOM = 3,           /* device allocation failed -> GpuRetryOOM                   */
  B2_ERR_SIZE_OVERFLOW = 4, /* > 2^31-1 rows / chars -> CudfColumnSizeOverflowException  */
  B2_ERR_UNSUPPORTED = 5,   /* would be tagged willNotWorkOnGpu by the plugin            */
  B2_ERR_FATAL = 6          /* CudaFatalException: executor must exit                    */
} b2_status;

/* Spark type -> cudf DType map of GpuColumnVector.java:417-453 */
typedef enum {
  B2_BOOL8 = 0,
  B2_INT8 = 1,
  B2_INT16 = 2,
  B2_INT32 = 3,
  B2_INT64 = 4,
  B2_FLOAT32 = 5,
  B2_FLOAT64 = 6,
  B2_DATE32 = 7,        /* TIMESTAMP_DAYS, int32 */
  B2_TIMESTAMP_US = 8,  /* TIMESTAMP_MICROSECONDS, int64 */
  B2_DECIMAL32 = 9,
  B2_DECIMAL64 = 10,
  B2_DECIMAL128 = 11,
  B2_STRING = 12
} b2_dtype;

typedef struct {
  int32_t dtype;        /* b2_dtype */
  int32_t scale;        /* Spark scale for decimals, else 0 */
  int64_t size;         /* rows */
  int64_t null_count;
  const void* data;     /* device pointer: values (fixed width) or chars (STRING) */
  const uint32_t* validity; /* device pointer or NULL when there are no nulls */
  const int32_t* offsets;   /* device pointer, STRING only */
  int64_t data_bytes;   /* bytes behind data */
} b2_column_info;

const char* b2_last_error(void);
const char* b2_version(void);

/* ---- runtime (Plugin.scala:599-702 RapidsExecutorPlugin.init; GpuDeviceManager.scala:397-445) --- */
int b2_init(int device, size_t pool_bytes);   /* Rmm.initialize analogue: stream-ordered pool */
int b2_shutdown(void);
int b2_stream_sync(void);                     /* Cuda.DEFAULT_STREAM.sync() */
int b2_set_stream(void* cuda_stream);         /* adopt the caller's stream for this thread */
void* b2_get_stream(void);
int b2_device_bytes_in_use(int64_t* out);
int b2_set_alloc_limit(int64_t bytes);        /* test hook: RmmSpark.forceRetryOOM analogue */

/* ---- (f4) memory pressure: spill store, semaphore, retry accounting ---------------------------------------------------------
 * SpillableColumnarBatch (spill/SpillFramework.scala:49-150): a batch held across iterator next() calls is registered here;
 * while nobody holds the table from b2_spillable_get the store may move it to host memory (on allocation failure, or on
 * b2_spill) and brings it back on the next get.  Allocation failure = spill, then B2_ERR_OOM (GpuRetryOOM): the exec layer
 * retries and, for joins and aggregates, splits the input batch and retries (RmmRapidsRetryIterator.scala:65-203). */
int b2_spillable_create(b2_handle table, b2_handle* out_spillable);
int b2_spillable_get(b2_handle spillable, b2_handle* out_table);     /* new reference; unspills when needed */
int b2_spillable_is_spilled(b2_handle spillable, int32_t* out);
int b2_spillable_close(b2_handle spillable);
int b2_spill(int64_t want_bytes, int64_t* out_freed);
/* out6: bytes in use, alloc limit, bytes spilled, bytes unspilled, retries, split-and-retries */
int b2_memory_stats(int64_t* out6);
/* GpuSemaphore (GpuSemaphore.scala:183-260): at most `permits` threads between acquire and release (0 = unlimited).
 * b2_exec_next acquires for the calling thread; the task releases when it is done with the GPU. */
int b2_semaphore_init(int32_t permits);
int b2_semaphore_acquire(void);
int b2_semaphore_release(void);
int b2_semaphore_stats(int64_t* out3);   /* permits, holders, times a thread had to wait */

/* ---- columns & tables (ai.rapids.cudf.ColumnVector / Table; GpuColumnVector.java:621-660) ------ */
/* host -> device (HostColumnarToGpu.scala, RapidsHostColumnBuilder + tryBuild H2D) */
int b2_column_from_host(int32_t dtype, int32_t scale, int64_t size, const void* data,
                        const uint8_t* validity_bits, const int32_t* offsets, b2_handle* out);
/* wrap-by-copy of device buffers the caller owns (e.g. a torch tensor) */
int b2_column_from_device(int32_t dtype, int32_t scale, int64_t size, const void* data,
                          const uint32_t* validity_bits, const int32_t* offsets, b2_handle* out);
int b2_column_info_get(b2_handle col, b2_column_info* out);
/* device -> host (ColumnVector.copyToHost; GpuColumnarToRowExec.scala:337-384) */
int b2_column_to_host(b2_handle col, void* data, uint8_t* validity_bits, int32_t* offsets);
int b2_column_incref(b2_handle col);
int b2_column_close(b2_handle col);
int b2_column_from_scalar(int32_t dtype, int32_t scale, int64_t size, const void* value16,
                          int32_t is_valid, b2_handle* out);   /* ColumnVector.fromScalar */

int b2_table_create(const b2_handle* cols, int32_t ncols, b2_handle* out);
int b2_table_num_rows(b2_handle table, int64_t* out);
int b2_table_num_columns(b2_handle table, int32_t* out);
int b2_table_column(b2_handle table, int32_t i, b2_handle* out); /* new reference */
int b2_table_incref(b2_handle table);
int b2_table_close(b2_handle table);

/* ---- a1: expression evaluation (GpuExpressions.scala:181 columnarEval, :197 convertToAst;
 *          basicPhysicalOperators.scala:116-140, 1052-1076 GpuTieredProject.project) ----------
 * An expression tree is built node by node (as GpuExpression.convertToAst builds cudf ast.*),
 * carries Spark types, and is compiled once into a register-machine program that ONE kernel
 * evaluates per batch (no per-node launch, no intermediate columns).                         */
typedef enum {
  /* arithmetic.scala:309-340 (Add/Subtract/Multiply), :411-640 decimal multiply */
  B2_OP_ADD = 1, B2_OP_SUB = 2, B2_OP_MUL = 3, B2_OP_DIV = 4, B2_OP_MOD = 5, B2_OP_PMOD = 6,
  B2_OP_NEG = 7, B2_OP_ABS = 8,
  /* predicates.scala:155-331 */
  B2_OP_EQ = 10, B2_OP_NE = 11, B2_OP_LT = 12, B2_OP_LE = 13, B2_OP_GT = 14, B2_OP_GE = 15,
  B2_OP_EQ_NULLSAFE = 16,
  /* predicates.scala:54-153 */
  B2_OP_AND = 20, B2_OP_OR = 21, B2_OP_NOT = 22,
  /* nullExpressions.scala */
  B2_OP_IS_NULL = 30, B2_OP_IS_NOT_NULL = 31, B2_OP_COALESCE = 32,
  /* conditionalExpressions.scala GpuIf */
  B2_OP_IF = 33,
  /* GpuCast.scala:295 doCast (numeric / decimal / date subset) */
  B2_OP_CAST = 40,
  /* NormalizeFloatingNumbers.scala:29-38 */
  B2_OP_NORMALIZE_NAN_ZERO = 41,
  /* datetimeExpressions.scala GpuYear */
  B2_OP_YEAR = 42,
  /* stringFunctions.scala:163 GpuStartsWith, :189 GpuEndsWith, :396 GpuContains, :972 GpuLike, :524 GpuSubstring.
   * String comparisons (EQ..GE) follow UTF8String.compareTo (unsigned bytes).  Strings are consumed by predicates;
   * a Substring is a window a predicate looks through (b2_substring materialises one as a column).            */
  B2_OP_STARTS_WITH = 50, B2_OP_ENDS_WITH = 51, B2_OP_CONTAINS = 52, B2_OP_LIKE = 53, B2_OP_SUBSTRING = 54
} b2_expr_op;

int b2_expr_column(int32_t index, int32_t dtype, int32_t precision, int32_t scale,
                   int32_t nullable, b2_handle* out);      /* GpuBoundReference */
/* literal: value is 16 bytes little endian (int/decimal sign-extended, double/float bits) */
int b2_expr_literal(int32_t dtype, int32_t precision, int32_t scale, const void* value16,
                    int32_t is_null, b2_handle* out);       /* GpuLiteral */
int b2_expr_unary(int32_t op, b2_handle child, b2_handle* out);
int b2_expr_binary(int32_t op, b2_handle left, b2_handle right, b2_handle* out);
int b2_expr_ternary(int32_t op, b2_handle a, b2_handle b, b2_handle c, b2_handle* out);
int b2_expr_cast(b2_handle child, int32_t dtype, int32_t precision, int32_t scale,
                 b2_handle* out);
int b2_expr_string_literal(const char* utf8, int32_t len, int32_t is_null, b2_handle* out); /* GpuLiteral(StringType) */
int b2_expr_like(b2_handle child, b2_handle pattern_literal, int32_t escape_char, b2_handle* out);   /* GpuLike */
int b2_expr_substring(b2_handle child, int32_t pos, int32_t len, b2_handle* out);  /* GpuSubstring, literal pos/len (1-based) */
/* GpuInSet.scala / In over a literal list: Kleene OR of equalities */
int b2_expr_in(b2_handle child, const b2_handle* literals, int32_t n, b2_handle* out);
/* conditionalExpressions.scala:322 GpuCaseWhen; else_value = 0 -> NULL */
int b2_expr_case_when(const b2_handle* conds, const b2_handle* values, int32_t n, b2_handle else_value,
                      b2_handle* out);
int b2_expr_type(b2_handle expr, int32_t* dtype, int32_t* precision, int32_t* scale,
                 int32_t* nullable);
int b2_expr_close(b2_handle expr);

/* compile N output expressions against an input schema into one program */
int b2_program_compile(const b2_handle* exprs, int32_t nexprs, b2_handle* out);
int b2_program_close(b2_handle program);
/* what a compiled program looks like to the kernels: instructions, registers, register bytes per row and rows per tile
 * (tile_rows / 256 rows per thread; the filter's TMA-staged and the group-by's fused kernels pick their own tile) */
int b2_program_info(b2_handle program, int32_t* ninstr, int32_t* nregs, int32_t* bytes_per_row, int32_t* tile_rows);
/* GpuProjectExec.project: table -> table of nexprs columns, one launch */
int b2_project(b2_handle program, b2_handle table, b2_handle* out_table);

/* GpuSubstring (stringFunctions.scala:524-620) with literal pos (1-based, negative = from the end) and len, materialised
 * as a new STRING column (code-point semantics of UTF8String.substringSQL) */
int b2_substring(b2_handle string_column, int32_t pos, int32_t len, b2_handle* out_column);

/* ---- a2: filter (basicPhysicalOperators.scala:1148-1224 GpuFilter; Table.filter(mask)) -------- */
int b2_filter_mask(b2_handle table, b2_handle bool_mask, b2_handle* out_table);
/* fused: predicate program (1 BOOL8 output) evaluated and compacted in one kernel */
int b2_filter(b2_handle predicate_program, b2_handle table, b2_handle* out_table);
/* GpuFilterExec under a column-pruning GpuProjectExec, fused: only keep_cols (in that order) are compacted */
int b2_filter_select(b2_handle predicate_program, b2_handle table, const int32_t* keep_cols, int32_t nkeep,
                     b2_handle* out_table);
/* selection vector of a filter: the INT32 row ids (ascending) of the rows that pass, nothing is compacted */
int b2_filter_row_ids(b2_handle predicate_program, b2_handle table, b2_handle* out_int32_ids);
/* count-only path, basicPhysicalOperators.scala:1161-1169 */
int b2_filter_count(b2_handle predicate_program, b2_handle table, int64_t* out_count);

/* ---- a3/a4/a5: aggregation (GpuAggregateExec.scala:540-585; aggregateFunctions.scala) ---------- */
typedef enum {
  B2_AGG_SUM = 1,      /* CudfSum; decimal sums use the Spark-exact 128-bit path (a5)     */
  B2_AGG_COUNT = 2,    /* CudfCount: non-null count -> INT64                               */
  B2_AGG_MIN = 3,
  B2_AGG_MAX = 4,
  B2_AGG_COUNT_ALL = 5,/* count(*)                                                         */
  B2_AGG_FIRST = 6,
  B2_AGG_ANY_VALID = 7 /* isEmpty flag of GpuDecimalSum: true iff no valid input (min(isNull)) */
} b2_agg_kind;

typedef struct {
  int32_t kind;        /* b2_agg_kind */
  int32_t column;      /* input column index in the table (ignored for COUNT_ALL) */
  int32_t out_dtype;   /* result dtype: e.g. B2_DECIMAL128 for sum(decimal64), INT64 for sum(int) */
  int32_t out_scale;
  int32_t out_precision; /* decimal sums: overflow of this precision -> NULL (GpuCheckOverflowAfterSum) */
} b2_agg_spec;

/* AggHelper.performReduction: one-row table, one column per spec; empty input -> null/0 */
int b2_reduce(b2_handle table, const b2_agg_spec* aggs, int32_t naggs, b2_handle* out_table);
/* AggHelper.performGroupByAggregation: keys first then aggregates; nulls form a group,
 * NaN==NaN, -0.0==0.0 (caller normalises);   output order unspecified                      */
int b2_groupby(b2_handle table, const int32_t* key_cols, int32_t nkeys,
               const b2_agg_spec* aggs, int32_t naggs, b2_handle* out_table);
/* fused scan: [filter] -> project -> reduce/groupby in one kernel.  The program's outputs are
 * the pre-step projection (GpuAggFirstPassIterator preStepBound); if has_predicate, output 0 is
 * the BOOL8 filter condition of the child GpuFilterExec and key/agg column indexes refer to the
 * remaining outputs.                                                                        */
int b2_scan_aggregate(b2_handle program, int32_t has_predicate, b2_handle table,
                      const int32_t* key_cols, int32_t nkeys,
                      const b2_agg_spec* aggs, int32_t naggs, b2_handle* out_table);
/* Table.distinctCount (GpuAggregateExec.scala:2177-2183; GpuHashJoin.scala:1015-1029) */
int b2_distinct_count(b2_handle table, const int32_t* key_cols, int32_t nkeys, int64_t* out);

/* ---- a6/a7: hash join (GpuHashJoin.scala:256-600, 1374-1553; JoinGatherer.scala:585-599) ------- */
typedef enum {
  B2_JOIN_INNER = 0, B2_JOIN_LEFT_OUTER = 1, B2_JOIN_LEFT_SEMI = 2, B2_JOIN_LEFT_ANTI = 3,
  B2_JOIN_FULL_OUTER = 4,
  /* every build row appears; stream columns NULL where no stream row matched.  Spark's RightOuter with BuildRight, and
   * LeftOuter with BuildLeft with the children swapped (the caller restores the column order with a bound-reference
   * projection) — HashOuterJoinIterator (GpuShuffledSizedHashJoinExec.scala:346-364, GpuHashJoin.scala:1807-1814) */
  B2_JOIN_RIGHT_OUTER = 5
} b2_join_kind;
/* build once per build batch (the reference rebuilds per stream batch: JoinPrimitives.hashInnerJoin
 * takes both key tables each call).  nulls_equal = compareNullsEqual (GpuHashJoin.scala:602-640) */
int b2_join_build(b2_handle build_keys_table, int32_t nulls_equal, b2_handle* out_hash_table);
int b2_join_hash_table_close(b2_handle ht);
/* probe: stream side is "left".  Returns INT32 gather-map columns (right map NULL for semi/anti).
 * For LEFT_OUTER unmatched rows carry INT32_MIN in the right map (OutOfBoundsPolicy.NULLIFY).
 * FULL_OUTER = the LEFT_OUTER maps followed by one row per build row that no stream row matched, in build order,
 * with INT32_MIN in the left map (Table.fullJoinGatherMaps; across stream batches the caller keeps the union of
 * matched build rows itself, as GpuHashJoin.scala's HashFullJoinIterator does).  RIGHT_OUTER = the INNER maps followed by
 * (INT32_MIN, b) for every build row b no stream row matched, ascending (through a selection vector too). */
int b2_join_probe(b2_handle ht, b2_handle probe_keys_table, int32_t kind,
                  b2_handle* out_left_map, b2_handle* out_right_map);
/* late materialisation: `selection` = INT32 row ids (ascending) of the stream rows that take part, e.g. the rows a
 * GpuFilterExec directly below the join keeps (b2_filter_row_ids); the left map carries ORIGINAL row ids, so the payload is
 * gathered from the unfiltered batch and the filtered copy is never written.  selection = 0: plain b2_join_probe. */
int b2_join_probe_sel(b2_handle ht, b2_handle probe_keys_table, b2_handle selection, int32_t kind,
                      b2_handle* out_left_map, b2_handle* out_right_map);
/* INNER join of the rows of `table` that pass `predicate_program` (a GpuFilterExec directly below the stream side).  When
 * the predicate is a conjunction of NOT NULL integer column-vs-literal comparisons and the build side is distinct on one
 * NOT NULL 4- or 8-byte integer key of the stream key's dtype, the filter is evaluated inside the probe kernel and no
 * selection vector exists; otherwise this is b2_filter_row_ids + b2_join_probe_sel.  key_col: the stream key's column in
 * `table`.  The left map carries ORIGINAL row ids of `table`; out_npass = rows that passed the filter. */
int b2_join_probe_filter(b2_handle ht, b2_handle table, int32_t key_col, b2_handle predicate_program,
                         b2_handle* out_left_map, b2_handle* out_right_map, int64_t* out_npass);
/* Matched build rows across stream batches, for outer joins that preserve the build side: a tracker is one bit per build row
 * of ONE hash table (zeroed at creation), kept apart from the table because a cached table is shared by task threads.
 * b2_join_probe_track = b2_join_probe_sel (kind INNER or LEFT_OUTER) that also sets the bit of every build row it finds,
 * inside the probe kernel (HashJoinStreamSideIterator.updateTrackingMask, GpuHashJoin.scala:2164-2204; the sub-partitioned
 * join keeps one per pair, GpuShuffledSizedHashJoinExec.scala:1760); a tracker of another table: B2_ERR_INVALID.
 * b2_join_tracker_mark sets the bits of right_map[i] where pass[i] (BOOL8, NULL = false; pass = 0: every i) — the pairs that
 * passed a join condition; negative entries are skipped, one >= the build row count gives B2_ERR_INVALID.  Marking is
 * idempotent.  b2_join_tracker_unmatched: ascending INT32 ids of the build rows never marked (HashOuterJoinIterator.getFinalBatch,
 * GpuHashJoin.scala:2288-2326). */
int b2_join_tracker_create(b2_handle ht, b2_handle* out_tracker);
int b2_join_tracker_close(b2_handle tracker);
int b2_join_probe_track(b2_handle ht, b2_handle probe_keys_table, b2_handle selection, int32_t kind, b2_handle tracker,
                        b2_handle* out_left_map, b2_handle* out_right_map);
int b2_join_tracker_mark(b2_handle tracker, b2_handle right_map, b2_handle pass);
int b2_join_tracker_unmatched(b2_handle tracker, b2_handle* out_ids);
/* Table.gather(map, OutOfBoundsPolicy): out-of-range index -> null row when nullify != 0 */
int b2_gather(b2_handle table, b2_handle int32_map, int32_t nullify_oob, b2_handle* out_table);

/* ---- a8: sort (SortUtils.scala:172-400; GpuSortExec.scala:87-165; limit.scala:234-330) --------- */
typedef struct {
  int32_t column;
  int32_t ascending;    /* 1 asc, 0 desc */
  int32_t nulls_first;  /* SortUtils.getOrder: asc(idx, nullsFirst) / desc(idx, nullsLast) */
} b2_order_by_arg;
int b2_sort_order(b2_handle table, const b2_order_by_arg* keys, int32_t nkeys,
                  b2_handle* out_int32_perm);                          /* Table.sortOrder (stable) */
int b2_order_by(b2_handle table, const b2_order_by_arg* keys, int32_t nkeys,
                b2_handle* out_table);                                 /* Table.orderBy */
int b2_top_n(b2_handle table, const b2_order_by_arg* keys, int32_t nkeys, int64_t n,
             b2_handle* out_table);                                    /* GpuTopN */
int b2_merge_sorted(const b2_handle* tables, int32_t ntables, const b2_order_by_arg* keys,
                    int32_t nkeys, b2_handle* out_table);              /* Table.merge */
/* Table.lowerBound / upperBound: for each row of `values`, its insertion index in sorted `table` */
int b2_search_bounds(b2_handle sorted_table, b2_handle values_table, const b2_order_by_arg* keys,
                     int32_t nkeys, int32_t upper, b2_handle* out_int32_idx);
/* GpuSortExec with the out-of-core sort (GpuSortExec.scala:130-165, GpuOutOfCoreSortIterator :241-630): a stable full sort
 * of the child's partition that need not fit on the device.  Sorted pieces wait in the spill store and are merged on the GPU;
 * output batches hold at most target_bytes (data + validity + offsets; raised to 16 KiB; a single row may be larger) and fewer
 * than 2^31 rows each. */
int b2_exec_sort_out_of_core(b2_handle child, const b2_order_by_arg* order, int32_t norder, int64_t target_bytes, b2_handle* out);

/* ---- a9: hash partition (HashFunctions.scala:196-209; GpuHashPartitioningBase.scala:36-110;
 *          GpuPartitioning.scala:66-99) ----------------------------------------------------------- */
int b2_murmur3(b2_handle table, const int32_t* cols, int32_t ncols, int32_t seed,
               b2_handle* out_int32_col);                              /* Hash.murmurHash32 */
/* murmur3(seed) pmod num_partitions, then Table.partition: rows reordered (stable) so each
 * partition is contiguous; offsets_out[num_partitions+1] (host) = partition starts */
int b2_hash_partition(b2_handle table, const int32_t* key_cols, int32_t nkeys, int32_t seed,
                      int32_t num_partitions, b2_handle* out_table, int32_t* offsets_out);
int b2_partition_by_ids(b2_handle table, b2_handle int32_part_ids, int32_t num_partitions,
                        b2_handle* out_table, int32_t* offsets_out);  /* Table.partition */
int b2_slice(b2_handle table, int64_t start, int64_t end, b2_handle* out_table); /* contiguousSplit piece */
/* GpuBatchSubPartitioner (GpuSubPartitionHashJoin.scala:86-221: hashPartition + contiguousSplit) in one pass: rows of `table`
 * (or only the rows of the INT32 selection vector `sel`, 0 = all rows) split into num_parts tables by
 * pmod(murmur3(key columns, seed), num_parts); each output owns its buffers, keeps the rows' input order and holds the columns
 * keep_cols (NULL = all, in that order); out_tables[p] = 0 when part p is empty.  2 <= num_parts <= 256. */
int b2_hash_split(b2_handle table, b2_handle sel, const int32_t* key_cols, int32_t nkeys, int32_t seed, int32_t num_parts,
                  const int32_t* keep_cols, int32_t nkeep, b2_handle* out_tables);

/* ---- a10: Parquet -> device (GpuParquetScan.scala:2089-2127 readPartFile, :3322-3503) ---------- */
/* host_buf is the reassembled mini-file "PAR1 + column chunks + footer + len + PAR1" exactly as
 * readPartFile builds it; columns are selected by name in output order (includeColumn order). */
int b2_parquet_decode(const uint8_t* host_buf, int64_t len, const char* const* column_names,
                      int32_t ncols, b2_handle* out_table);
/* same, but the file bytes are already resident in device memory (bench `value` leg) */
int b2_parquet_decode_device(const uint8_t* host_buf, const uint8_t* dev_buf, int64_t len,
                             const char* const* column_names, int32_t ncols, b2_handle* out_table);

/* one task's split of the file: only row groups [rg_begin, rg_end) are decoded (GpuParquetScan.scala filterBlocks /
 * clipBlocksToSchema: a Spark task reads the row groups of its input split); dev_buf may be NULL (bytes on the host) */
int b2_parquet_decode_row_groups(const uint8_t* host_buf, const uint8_t* dev_buf, int64_t len,
                                 const char* const* column_names, int32_t ncols, int32_t rg_begin, int32_t rg_end,
                                 b2_handle* out_table);
int b2_parquet_num_row_groups(const uint8_t* host_buf, int64_t len, int32_t* out_count);
/* ai.rapids.cudf.ParquetChunkedReader (GpuParquetScan.scala:3403-3407, 3497-3498): decode the buffer in chunks whose decoded
 * size stays under chunk_byte_limit (0 = no byte limit) and under 2^31-1 rows; a chunk is a run of whole row groups.
 * host_buf must outlive the reader. */
int b2_parquet_chunked_open(const uint8_t* host_buf, int64_t len, const char* const* column_names, int32_t ncols,
                            int64_t chunk_byte_limit, b2_handle* out_reader);
int b2_parquet_chunked_has_next(b2_handle reader, int32_t* out);
int b2_parquet_chunked_next(b2_handle reader, b2_handle* out_table);
int b2_parquet_chunked_close(b2_handle reader);

/* byte accounting of this thread's last decode (roofline numerators of bench.py):
 * out[0] compressed bytes fed to the decompressor, out[1] bytes it produced, out[2] uncompressed
 * bytes of all data+dictionary pages, out[3] bytes of the output columns, out[4] pages */
int b2_parquet_last_stats(int64_t* out5);

/* ---- a11: row <-> column (GpuColumnarToRowExec.scala:44-220 RowConversion.convertToRows*;
 *           GpuRowToColumnarExec.scala:574-755) -------------------------------------------------- */
/* JCUDF fixed-width row format: columns packed in order at natural alignment, then validity
 * bytes (1 bit per column), row padded to 8 B.  Returns row size; rows written to host_rows. */
int b2_rows_size(b2_handle table, int32_t* row_bytes);
int b2_table_to_rows(b2_handle table, uint8_t* host_rows, int64_t capacity_bytes);
int b2_table_from_rows(const uint8_t* host_rows, int64_t nrows, const int32_t* dtypes,
                       const int32_t* scales, int32_t ncols, b2_handle* out_table);

/* ---- a12: concatenate (GpuAggregateExec.scala:700-727; GpuCoalesceBatches.scala:43-108) -------- */
int b2_concat(const b2_handle* tables, int32_t ntables, b2_handle* out_table);

/* ---- (f1) shuffle wire format + coalesce on read (GpuColumnarBatchSerializer.scala:169-320, 385-470;
 *      GpuShuffleCoalesceExec.scala:72-110, 371-475).  Format "B2T1" (serialize.cu): header, per-column descriptors, then
 *      validity / offsets / data buffers padded to 64 bytes — the structure of JCudfSerialization's header + host buffer. */
int b2_serialized_size(b2_handle table, int64_t row_start, int64_t row_end, int64_t* out_bytes);
int b2_serialize_table(b2_handle table, int64_t row_start, int64_t row_end, uint8_t* host_out, int64_t capacity,
                       int64_t* out_written);
/* N serialised tables -> one device table: concatenated on the host, one upload per column buffer */
int b2_deserialize_concat(const uint8_t* const* bufs, const int64_t* lens, int32_t nbufs, b2_handle* out_table);

/* ---- (e) exchange: RapidsShuffleManager replaced by NCCL all-to-all over NVLink ---------------
 * (GpuShuffleExchangeExecBase.scala:384-536; RapidsShuffleInternalManagerBase.scala:1618, 1978) */
int b2_comm_unique_id(uint8_t* out128);                       /* ncclGetUniqueId (rank 0) */
int b2_comm_init(const uint8_t* id128, int32_t rank, int32_t world, b2_handle* out_comm);
int b2_comm_close(b2_handle comm);
/* table is already partitioned: offsets[world+1] (host) delimit the rows for each rank.  Returns
 * the concatenation of what every rank sent to me. */
int b2_exchange(b2_handle comm, b2_handle partitioned_table, const int32_t* offsets,
                b2_handle* out_table);
/* same with the termination protocol of GpuShuffleExchangeExec: partitioned_table = 0 (offsets NULL) when this rank has no
 * batch for this call; *any_data = some rank had one (0: the exchange is over everywhere, *out_table = 0) */
int b2_exchange_ex(b2_handle comm, b2_handle partitioned_table, const int32_t* offsets,
                   b2_handle* out_table, int32_t* any_data);
/* FUSED GpuHashPartitioning + shuffle write + read for fixed-width tables: one kernel hashes the keys (Spark Murmur3 pmod
 * world; nkeys = 0: SinglePartition -> rank 0) and stores every row straight into the destination GPU's receive arena
 * over NVLink peer mappings; one 400-byte header all-gather is the size exchange and the completion barrier.
 * (GpuShuffleExchangeExecBase.scala:384-536, GpuHashPartitioningBase.scala:36-54, GpuPartitioning.scala:66-99) */
int b2_exchange_hash(b2_handle comm, b2_handle table, const int32_t* key_cols, int32_t nkeys, int32_t seed,
                     b2_handle* out_table, int32_t* any_data);
/* same through a selection vector (see b2_join_probe_sel): only rows `selection` names are sent, and only columns out_cols
 * (a filter + column pruning directly below the exchange, fused into the scatter) */
int b2_exchange_hash_sel(b2_handle comm, b2_handle table, b2_handle selection, const int32_t* out_cols, int32_t nout,
                         const int32_t* key_cols, int32_t nkeys, int32_t seed, b2_handle* out_table, int32_t* any_data);
int b2_comm_fused_ready(b2_handle comm, int32_t* ok);        /* collective: peer arenas mapped on every rank? */
int b2_comm_allmax(b2_handle comm, int32_t value, int32_t* out);   /* collective max of one int per rank */
/* GpuShuffleExchangeExec termination without an empty last round: `more` = this rank will call the next exchange with a batch
 * (it looked one batch ahead); after the call b2_comm_any_more tells whether any rank will.  Unset: more = "had data". */
int b2_comm_set_more(b2_handle comm, int32_t more);
int b2_comm_any_more(b2_handle comm, int32_t* out);
/* out4: payload bytes sent to / received from OTHER ranks so far, exchange calls, arena bytes (0 = NCCL path) */
int b2_comm_stats(b2_handle comm, int64_t* out4);
/* GpuBroadcastExchangeExec data movement: root's table to every rank (ncclBroadcast); non-root pass table = 0 */
int b2_broadcast_table(b2_handle comm, b2_handle table, int32_t root, b2_handle* out_table);

/* ---- host operator layer: C++ mirror of the GpuExec nodes of the hot path (exec.cu).  Every node is
 * a pull iterator of batches — GpuExec.internalDoExecuteColumnar(): RDD[ColumnarBatch]
 * (GpuExec.scala:106,190,380).  b2_exec_next returns 0 in *out_table when the node is exhausted. */
int b2_exec_source(b2_handle* out);                                   /* child RDD stand-in */
int b2_exec_source_push(b2_handle source, b2_handle table);
/* HostColumnarToGpu (HostColumnarToGpu.scala): host columnar batches -> device, the copy of batch k+1 overlapping the
 * consumption of batch k.  The host buffers (pinned for full PCIe speed) must outlive the node. */
typedef struct {
  int32_t dtype, scale;
  int64_t rows;
  const void* data;              /* values, or chars for STRING */
  const uint8_t* validity_bits;  /* NULL = no nulls */
  const int32_t* offsets;        /* STRING: rows + 1 offsets */
} b2_host_column;
int b2_exec_host_source(b2_handle* out);
int b2_exec_host_source_push(b2_handle source, const b2_host_column* cols, int32_t ncols);
int b2_exec_parquet_scan(const char* const* column_names, int32_t ncols, b2_handle* out);      /* GpuParquetScan.scala:3543-3600 */
int b2_exec_parquet_scan_add(b2_handle scan, const uint8_t* host_buf, int64_t len);            /* buffer must outlive the scan */
int b2_exec_filter(b2_handle child, b2_handle predicate_program, b2_handle* out);              /* GpuFilterExec :1238-1291 */
/* GpuProjectExec(column pruning) over GpuFilterExec, fused: only keep_cols are compacted */
int b2_exec_filter_select(b2_handle child, b2_handle predicate_program, const int32_t* keep_cols, int32_t nkeep, b2_handle* out);
int b2_exec_project(b2_handle child, b2_handle program, b2_handle* out);                       /* GpuProjectExec :755-884 */
/* GpuExpandExec (GpuExpandExec.scala): each batch projected once per projection list, results stacked (GROUPING SETS,
 * several COUNT(DISTINCT)); all projection programs must produce the same output types */
int b2_exec_expand(b2_handle child, const b2_handle* projection_programs, int32_t nprojections, b2_handle* out);
/* GpuHashAggregateExec (GpuAggregateExec.scala:1942-2085).  PARTIAL and COMPLETE update the aggregates over
 * the program's outputs; FINAL merges aggregation buffers.  A buffer (PARTIAL's output, FINAL's input) is the
 * keys, one column per aggregate, then one INT64 count of valid inputs per decimal SUM, in aggregate order
 * (Spark's isEmpty): a NULL partial sum with a nonzero count overflowed, and makes the merged sum NULL. */
typedef enum { B2_AGG_MODE_PARTIAL = 0, B2_AGG_MODE_FINAL = 1, B2_AGG_MODE_COMPLETE = 2 } b2_agg_mode;
int b2_exec_hash_aggregate(b2_handle child, b2_handle program, int32_t has_predicate, int32_t mode,
                           const int32_t* keys, int32_t nkeys, const b2_agg_spec* aggs, int32_t naggs, b2_handle* out);
/* GpuMergeAggregateIterator repartitioning (GpuAggregateExec.scala:150-307, 863-1103), for partial results larger than the
 * device.  Every piece (a first-pass partial; in FINAL mode an input batch) is held in the spill store.  When the held bytes
 * (table_bytes) pass target_bytes they are merged into one; a result of at most target_bytes / 2 stays the only held piece,
 * a larger one is split by murmur3 seed 107 of the keys into num_buckets (2..256; Spark default 16) spillable buckets, and
 * so is every later piece.  A bucket still over the target is split again with seed 107 + 7 * depth, down to depth 10, and
 * then merged as it is; otherwise adjacent buckets are taken while they stay within the target and merged into one output
 * batch.  Memory: at most target_bytes of partials per merge (except a bucket at depth 10), plus that merge's workspace;
 * the rows of a single key must fit on the device.  Output rows and batches differ from the single merge's in order only.
 * Without this call, on a keyless aggregate (accepted, no effect), or when the held pieces never pass the target, the node
 * is unchanged.  B2_ERR_INVALID: target_bytes <= 0, num_buckets outside 2..256, not an aggregate, or already running. */
int b2_exec_aggregate_set_repartitioning(b2_handle agg, int64_t target_bytes, int32_t num_buckets);
/* out4: first-level buckets (0 = never bucketed), buckets split again, bytes split over all levels, deepest level reached */
int b2_exec_aggregate_repartition_stats(b2_handle agg, int64_t* out4);
/* GpuShuffledHashJoinExec (GpuShuffledHashJoinExec.scala:228-385): output = stream columns ++ build columns.  RIGHT_OUTER joins
 * the stream batches one at a time, tracking the build rows found (b2_join_probe_track), and after the last one emits the
 * unmatched build rows with NULL stream columns, in batches halved until they fit; no stream batch at all, or no build
 * batch: B2_ERR_UNSUPPORTED.  FULL_OUTER without a condition coalesces the stream side into one batch. */
int b2_exec_shuffled_hash_join(b2_handle stream_child, b2_handle build_child, const int32_t* stream_keys,
                               const int32_t* build_keys, int32_t nkeys, int32_t kind, int32_t nulls_equal, b2_handle* out);
/* same with a column-pruning GpuProjectExec above the join fused into the gathers: output = stream_out ++ build_out */
int b2_exec_shuffled_hash_join_select(b2_handle stream_child, b2_handle build_child, const int32_t* stream_keys,
                                      const int32_t* build_keys, int32_t nkeys, int32_t kind, int32_t nulls_equal,
                                      const int32_t* stream_out, int32_t nstream_out, const int32_t* build_out,
                                      int32_t nbuild_out, b2_handle* out);
/* mixed join: an extra non-equi condition (BOOL8 program bound over [stream columns ++ build columns]) decides which
 * equi-matched pairs survive — Table.mixed{Inner,Left,LeftSemi,LeftAnti}JoinGatherMap(s) (GpuHashJoin.scala:335-600),
 * ConditionalHashJoinIterator (:1556).  Inner / left outer / left semi / left anti / right outer / full outer; right outer and
 * full outer mark the build rows of the passing pairs in a tracker and emit the others after the last stream batch. */
int b2_exec_join_set_condition(b2_handle join, b2_handle condition_program);
/* GpuSubPartitionHashJoin (GpuShuffledHashJoinExec.scala:228-281, GpuSubPartitionHashJoin.scala:86-617): when the build side
 * passes target_bytes (table_bytes; raised to 16 KiB) both sides are split into num_partitions (2..256; Spark default 16,
 * RapidsConf.scala:2660) spillable buckets by murmur3 seed 100 of the join keys and joined bucket by bucket; adjacent small
 * buckets are packed up to the target, a bucket still over it (FULL OUTER without a condition: by its build or its stream
 * side) is split once
 * more (seed 110) and then joined as it is, so the rows of a single key must fit on the device.  Without this call, or when the build side stays within target_bytes,
 * the join is unchanged. */
int b2_exec_join_set_sub_partitioning(b2_handle join, int64_t target_bytes, int32_t num_partitions);
/* out4: first-level buckets (0 = not sub-partitioned), buckets repartitioned, build bytes split, stream bytes split */
int b2_exec_join_sub_partition_stats(b2_handle join, int64_t* out4);
/* out3: stream batches whose output rows the filter-probe kernel wrote (the emitting probe of an INNER FK -> PK join with a
 * simple filter below its stream side), batches joined through gather maps, and emitted batches whose matches passed the
 * estimated output size and were joined again through the maps (counted among the maps batches as well) */
int b2_exec_join_emit_stats(b2_handle join, int64_t* out3);
/* GpuBroadcastExchangeExec (GpuBroadcastExchangeExec.scala): every rank gets the whole child relation, one batch.  Used as
 * the build child of a join it makes GpuBroadcastHashJoinExec (GpuBroadcastHashJoinExecBase.scala:1-203). */
int b2_exec_broadcast_exchange(b2_handle child, b2_handle comm, int32_t rank, int32_t world, b2_handle* out);
/* GpuSortExec (global != 0: full sort, else each batch) / GpuTopN when limit >= 0 */
int b2_exec_sort(b2_handle child, const b2_order_by_arg* order, int32_t norder, int32_t global, int64_t limit, b2_handle* out);
int b2_exec_coalesce(b2_handle child, int64_t target_rows, b2_handle* out);                    /* GpuCoalesceBatches */
/* GpuShuffleExchangeExec: hash partition on key_cols (none = SinglePartition) + NCCL all-to-all */
int b2_exec_shuffle_exchange(b2_handle child, const int32_t* key_cols, int32_t nkeys, b2_handle comm, int32_t world, b2_handle* out);
int b2_exec_next(b2_handle exec, b2_handle* out_table);
int b2_exec_metrics(b2_handle exec, int64_t* out3);  /* numOutputRows, numOutputBatches, opTime (ns) */
/* device time of the node while b2_profile_enable(1) was on: out2[0] = self ms (children pulled from inside next() excluded),
 * out2[1] = total ms */
int b2_exec_device_time(b2_handle exec, double* out2);
int b2_exec_close(b2_handle exec);

/* ---- timing hooks for bench.py (CUDA events on the library stream) ------------------------------ */
int b2_event_create(b2_handle* out);
int b2_event_record(b2_handle ev);
int b2_event_elapsed_ms(b2_handle start, b2_handle stop, float* ms);
int b2_event_close(b2_handle ev);
int b2_kernel_launch_count(int64_t* out);   /* number of kernels this library launched so far */
/* per-kernel device time (CUDA events around each launch on the library stream), for the roofline
 * line of bench.py.  report: JSON array [{"name":..,"launches":n,"ms":total}] written to buf. */
int b2_profile_enable(int32_t on);
int b2_profile_report(char* buf, int64_t capacity);
/* pin / unpin caller memory for fast H2D (HostAlloc.scala pinned pool analogue) */
int b2_host_register(void* ptr, int64_t bytes);
int b2_host_unregister(void* ptr);
/* raw device buffer (bench: Parquet bytes resident in HBM) */
int b2_device_alloc(int64_t bytes, void** out);
int b2_device_free(void* ptr);
int b2_memcpy_h2d(void* dst, const void* src, int64_t bytes);
/* asynchronous staging of a host buffer on a dedicated copy stream, so the H2D of the next scan batch
 * overlaps the decode of the current one (what the reference's multithreaded Parquet reader does with
 * its host buffers: GpuMultiFileReader.scala).  b2_upload_wait orders the calling thread's compute
 * stream after the copy without blocking the host. */
int b2_upload_start(const void* pinned_host, int64_t bytes, b2_handle* out_upload);
int b2_upload_wait(b2_handle upload, void** out_device_ptr);
int b2_upload_free(b2_handle upload);

#if defined(__GNUC__)
#pragma GCC visibility pop
#endif
#ifdef __cplusplus
}
#endif
#endif /* B200SQL_H */
