/*
 * gsql_gpu.h — C ABI of the H100-native MPP operator hot path for GalaxySQL (PolarDB-X CN).
 *
 * This is the drop-in boundary: exactly the entry points a JNI shim under
 * com.alibaba.polardbx.executor.operator.Gpu*Exec would bind (INTEGRATION.md shows the Java/JNI side).
 * Plain pointers and sizes only; no CUDA, torch or C++ types in any signature.
 *
 * Reference interfaces replaced (paths relative to
 * polardbx-executor/src/main/java/com/alibaba/polardbx/executor/):
 *   gsql_batch / gsql_col        <- chunk/Chunk.java:41-100, chunk/Block.java:33, chunk/AbstractBlock.java:27-47
 *                                   (IntegerBlock.java:37 int[], LongBlock.java:41 long[], DoubleBlock.java:33 double[],
 *                                    boolean[] isNull -> one byte per row)
 *   gsql_hash_rows               <- chunk/Chunk.java:116-130 (hashCodeVector / hashCode)
 *   gsql_partition_ids           <- utils/ExecUtils.java:1023-1031 (partition)
 *   gsql_join_*                  <- operator/ParallelHashJoinExec.java:64-85 (ctor), :157-166 (consumeChunk),
 *                                   :107-128 (buildConsume), operator/AbstractBufferedJoinExec.java:116-264
 *                                   (doNextChunk / nextRows), :168-201 (nextJoinNullRows)
 *   gsql_agg_*                   <- operator/HashAggExec.java:74-91 (ctor), :133-145 (consumeChunk), :158-162
 *                                   (buildConsume), operator/AbstractHashAggExec.java:57-63 (doNextChunk)
 *   gsql_xchg_*                  <- mpp/operator/PartitioningExchanger.java:71-135 (local exchange),
 *                                   mpp/operator/PartitionedOutputCollector.java:170-196 + ExchangeClient.java:62-548
 *                                   (remote shuffle; replaced by an NCCL AllToAllv over NVLink)
 *
 * Threading: every handle is thread-compatible (the caller serialises calls on one handle, as the reference's
 * Driver does — mpp/operator/Driver.java:449-508); distinct handles may be used from distinct threads.
 * Errors: every call returns a gsql_status; gsql_last_error(ctx) gives the message.  CUDA/NCCL errors are sticky
 * per context.  *_destroy never fails and accepts NULL.
 * There is NO CPU fallback anywhere behind this ABI: without a CUDA device gsql_ctx_create fails with GSQL_E_CUDA.
 */
#ifndef GSQL_GPU_H
#define GSQL_GPU_H

#include <stddef.h>
#include <stdint.h>

#ifdef __cplusplus
extern "C" {
#endif
#if defined(__GNUC__)
#pragma GCC visibility push(default) /* the library is built with -fvisibility=hidden: only this ABI is exported */
#endif

#define GSQL_ABI_VERSION 1
#define GSQL_MAX_KEYS 8
#define GSQL_MAX_COLS 32
#define GSQL_MAX_AGGS 16
#define GSQL_MAX_PARTS 1024

typedef enum gsql_status {
    GSQL_OK = 0,
    GSQL_E_INVALID = 1,           /* bad argument / unsupported combination (planner must fall through) */
    GSQL_E_CUDA = 2,
    GSQL_E_NCCL = 3,
    GSQL_E_CAPACITY = 4,          /* output buffer too small; *out_rows holds the required row count */
    GSQL_E_MORE_THAN_ONE_ROW = 5, /* ErrorCode.ERR_SCALAR_SUBQUERY_RETURN_MORE_THAN_ONE_ROW */
    GSQL_E_UNSUPPORTED = 6,
    GSQL_E_STATE = 7,             /* call order violated (e.g. probe before build_finish) */
    GSQL_E_OOM = 8
} gsql_status;

typedef enum gsql_type {
    GSQL_T_INT32 = 0,  /* IntegerBlock */
    GSQL_T_INT64 = 1,  /* LongBlock    */
    GSQL_T_FP64 = 2,   /* DoubleBlock  */
    GSQL_T_DEC128 = 3  /* output only: exact SUM(int|bigint) as a little-endian two's-complement int128, scale 0
                          (stands for the DECIMAL of LittleNum2DecimalSum.java:45-82) */
} gsql_type;

typedef enum gsql_mem { GSQL_MEM_HOST = 0, GSQL_MEM_DEVICE = 1 } gsql_mem;

typedef enum gsql_join_type {
    GSQL_JOIN_INNER = 0, GSQL_JOIN_LEFT = 1, GSQL_JOIN_RIGHT = 2, GSQL_JOIN_SEMI = 3, GSQL_JOIN_ANTI = 4
} gsql_join_type;

typedef enum gsql_agg_kind {
    GSQL_AGG_COUNT_STAR = 0, /* CountRow */
    GSQL_AGG_COUNT = 1,      /* Count: all listed columns non-NULL */
    GSQL_AGG_SUM = 2,        /* FP64 -> FP64 (Double2DoubleSum); INT32/INT64 -> DEC128 (Int/Long2DecimalSum) */
    GSQL_AGG_AVG = 3,        /* FP64 -> FP64 (Double2DoubleAvg) */
    GSQL_AGG_MIN = 4,
    GSQL_AGG_MAX = 5,
    GSQL_AGG_SUM0 = 6,       /* INT64 -> INT64 wrapping, never NULL (Long2LongSum0) */
    GSQL_AGG_AVG_MERGE = 7,  /* final stage of a two-phase AVG(double): cols = {partial SUM (FP64), partial COUNT (BIGINT)};
                                result = sum of sums / (double) sum of counts, NULL when the counts add up to 0 — the
                                global SUM + global COUNT + DIVIDE project of CBOPushAggRule.splitAgg:256-310 in one call */
    GSQL_AGG_FIRST_VALUE = 8, /* InternalFirstValue (__FIRST_VALUE): one column, INT32 / INT64 / FP64 -> the same type, bits
                                unchanged (a NaN keeps its payload, -0.0 stays -0.0).
                                gsql_agg: a group's value is that of the first row accumulated into it, NULL included; first
                                = earliest consume call, then lowest row position within the batch as passed.  When the
                                aggregation ends with exactly one group (always so without group keys) the value is instead
                                the first non-NULL one of that group, NULL if there is none or no row at all.  Rows are
                                ordered by a 64-bit tag: consume ordinal (27 bits) | row position (36 bits) | NULL (1 bit);
                                a consume call beyond 2^27 - 2 or a batch of 2^36 rows or more is GSQL_E_CAPACITY.
                                gsql_sortagg: every group's first non-NULL value, NULL if all are NULL (SortAggExec resets
                                the aggregator per group, so the one-group rule always applies).
                                A FILTER argument (filter_arg >= 0) is GSQL_E_UNSUPPORTED on both: the stock aggregator
                                loses its place when a group's first row is filtered out. */
    /* Window functions: gsql_window only (gsql_agg_create and gsql_sortagg_create refuse them as unknown kinds). */
    GSQL_AGG_ROW_NUMBER = 9,  /* RowNumber: no columns; BIGINT, never NULL */
    GSQL_AGG_RANK = 10,       /* Rank: 0..4 peer columns; BIGINT, never NULL */
    GSQL_AGG_DENSE_RANK = 11  /* DenseRank: 0..4 peer columns; BIGINT, never NULL */
} gsql_agg_kind;

/* One Block.  `nulls` == NULL means "no NULLs" (AbstractBlock.mayHaveNull() == false); otherwise one byte per
 * row, non-zero = NULL, exactly the reference's boolean[] isNull. */
typedef struct gsql_col {
    int32_t type;     /* gsql_type */
    int32_t reserved;
    void *data;
    uint8_t *nulls;
} gsql_col;

/* One Chunk (or many concatenated chunks: the GPU operators want large batches). All pointers of a batch live in
 * the same memory space `mem`.  Host pointers should come from gsql_host_alloc (pinned) for full PCIe speed. */
typedef struct gsql_batch {
    int64_t rows;
    int32_t ncols;
    int32_t mem; /* gsql_mem */
    gsql_col *cols;
} gsql_batch;

typedef struct gsql_ctx gsql_ctx;
typedef struct gsql_join gsql_join;
typedef struct gsql_agg gsql_agg;
typedef struct gsql_xchg gsql_xchg;

/* ------------------------------------------------------------------------------------------------ context */
int gsql_abi_version(void);
gsql_status gsql_ctx_create(int device, gsql_ctx **out);
void gsql_ctx_destroy(gsql_ctx *ctx);
const char *gsql_last_error(const gsql_ctx *ctx);
gsql_status gsql_ctx_sync(gsql_ctx *ctx);
/* The CUDA stream (cudaStream_t as void*) every kernel of this context is launched on; callers that keep data
 * device-resident order their own work against it. */
void *gsql_ctx_stream(gsql_ctx *ctx);
gsql_status gsql_ctx_set_stream(gsql_ctx *ctx, void *cuda_stream);
/* Per-kernel device timing (CUDA events on the launching stream).  Off by default. */
gsql_status gsql_ctx_profile(gsql_ctx *ctx, int enable);
gsql_status gsql_ctx_profile_reset(gsql_ctx *ctx);
/* Returns launches and total milliseconds of kernel `name` since the last reset (synchronises the stream). */
gsql_status gsql_ctx_profile_get(gsql_ctx *ctx, const char *name, int64_t *launches, double *total_ms);
/* Writes up to `cap` bytes of "name launches ms\n" lines; returns the number of kernels recorded. */
int gsql_ctx_profile_dump(gsql_ctx *ctx, char *buf, size_t cap);
/* Total number of kernels this library launched on this context since creation. */
int64_t gsql_ctx_launch_count(const gsql_ctx *ctx);

gsql_status gsql_host_alloc(size_t bytes, void **out); /* pinned host memory */
void gsql_host_free(void *p);
gsql_status gsql_device_alloc(gsql_ctx *ctx, size_t bytes, void **out);
void gsql_device_free(gsql_ctx *ctx, void *p);
gsql_status gsql_memcpy_h2d(gsql_ctx *ctx, void *dst, const void *src, size_t bytes);
gsql_status gsql_memcpy_d2h(gsql_ctx *ctx, void *dst, const void *src, size_t bytes);

/* ------------------------------------------------------------------------------------------------ hashing */
/* out[r] = Chunk.hashCode over key_cols[0..nkeys) converted to unified_types (NULL -> 0, h = h*31 + c).
 * `out` lives in batch->mem.  Bit-exact with the reference (and with the oracle). */
gsql_status gsql_hash_rows(gsql_ctx *ctx, const gsql_batch *batch, const int32_t *key_cols, int32_t nkeys,
                           const int32_t *unified_types, int32_t *out);
/* out[r] = ExecUtils.partition(hash[r], nparts).  `mem` says where hash/out live. */
gsql_status gsql_partition_ids(gsql_ctx *ctx, const int32_t *hash, int64_t rows, int32_t nparts, int32_t *out,
                               int32_t mem);

/* ------------------------------------------------------------------------------------------------ hash join */
typedef struct gsql_join_spec {
    int32_t join_type;   /* gsql_join_type */
    int32_t max_one_row; /* singleJoin: output = outer cols + first inner col; 2nd match is an error */
    int32_t build_outer; /* buildOuterInput: the outer side is the build side */
    int32_t nkeys;
    int32_t outer_key[GSQL_MAX_KEYS]; /* EquiJoinKey.outerIndex */
    int32_t inner_key[GSQL_MAX_KEYS]; /* EquiJoinKey.innerIndex */
    int32_t key_type[GSQL_MAX_KEYS];  /* EquiJoinKey.unifiedType; keys match by value in it, a DOUBLE by its bits:
                                         -0.0 matches only -0.0, NaN matches nothing, a NULL component matches nothing */
    int32_t n_outer_cols;
    int32_t outer_types[GSQL_MAX_COLS];
    int32_t n_inner_cols;
    int32_t inner_types[GSQL_MAX_COLS];
    int32_t n_anti_operands;          /* 0 = antiJoinOperands == null (NOT EXISTS); else NOT IN null rules */
    int32_t anti_operands[GSQL_MAX_KEYS];
    /* otherCondition, restricted form: AND_i (joinRow[cond_col[i]] IS NULL OR joinRow[cond_col[i]] != cond_ne_value[i])
     * over integer columns of the join row (leftSide || rightSide).  n_cond == 0 <=> otherCondition == null. */
    int32_t n_cond;
    int32_t cond_col[4];
    int64_t cond_ne_value[4];
    int64_t expected_build_rows; /* hint, 0 = unknown */
} gsql_join_spec;

typedef struct gsql_join_info {
    int64_t build_rows;
    int64_t table_slots;
    int64_t table_bytes;
    int64_t device_bytes; /* everything the handle holds in HBM */
    int32_t has_duplicate_keys;
    int32_t pass_through; /* 1: probe rows pass unchanged (ANTI with empty build) */
    int32_t pass_nothing; /* 1: no output at all */
    int32_t fast_path;    /* 1: single integer key specialisation active */
    int32_t partitions;   /* >1: radix-partitioned (L2-resident) probe */
    int32_t reserved;
} gsql_join_info;

gsql_status gsql_join_create(gsql_ctx *ctx, const gsql_join_spec *spec, gsql_join **out);
/* consumeChunk on the build side: appends (copies) the batch; nothing of `batch` is referenced after return. */
gsql_status gsql_join_build_consume(gsql_join *j, const gsql_batch *build_rows);
/* Zero-copy variant for a device-resident build side that arrives as ONE batch (the output of an exchange or of
 * another GPU operator): the columns are referenced, not copied — exactly the reference's ownership rule (the consumer
 * retains consumed chunks: operator/util/ChunksIndex.java:48-51).  The batch must stay valid and unchanged until
 * gsql_join_destroy; no other build batch may be consumed on this handle. */
gsql_status gsql_join_build_consume_ref(gsql_join *j, const gsql_batch *build_rows);
/* buildConsume: builds the hash table over everything consumed. */
gsql_status gsql_join_build_finish(gsql_join *j);
gsql_status gsql_join_info_get(gsql_join *j, gsql_join_info *info);
/* Output schema (AbstractJoinExec.java:103-120). */
gsql_status gsql_join_output_schema(gsql_join *j, int32_t *ncols, int32_t *types /* GSQL_MAX_COLS*2 */);
/* Number of output rows `probe` would produce (exact). */
gsql_status gsql_join_probe_count(gsql_join *j, const gsql_batch *probe, int64_t *out_rows);
/* nextChunk over a probe batch.  `out` must be in probe->mem, with out->ncols columns of the output schema and
 * room for `out_capacity` rows; a column whose `nulls` is NULL must not receive a NULL (else GSQL_E_INVALID).
 * On GSQL_E_CAPACITY *out_rows is the required capacity.  Row order is unspecified (the reference's is too:
 * BaseExecTest.java:78-103 compares multisets). */
gsql_status gsql_join_probe(gsql_join *j, const gsql_batch *probe, gsql_batch *out, int64_t out_capacity,
                            int64_t *out_rows);
/* build_outer only, after the last probe: the unmatched build rows, NULL-padded (nextJoinNullRows). */
gsql_status gsql_join_unmatched_build(gsql_join *j, gsql_batch *out, int64_t out_capacity, int64_t *out_rows);
void gsql_join_destroy(gsql_join *j);

/* ------------------------------------------------------------------------------------------------ hash agg */
typedef struct gsql_agg_call {
    int32_t kind; /* gsql_agg_kind */
    int32_t ncols;
    int32_t cols[4];
    int32_t filter_arg; /* -1 = none (AggregateCall.filterArg) */
} gsql_agg_call;

/* Fused scan-side Project / Filter (the restricted forms TPC-H Q1 / Q3 need; replaces a VectorizedProjectExec /
 * VectorizedFilterExec directly under the HashAgg — operator/VectorizedProjectExec.java:40-143).  A derived column is
 * an FP64 value computed per row from FP64/INT input columns; it is NULL when any operand is NULL.  Aggregate calls
 * address derived column i as column index n_input_cols + i. */
typedef enum gsql_expr_kind {
    GSQL_EXPR_MUL_1MINUS = 1,        /* a * (1 - b)            e.g. l_extendedprice * (1 - l_discount) */
    GSQL_EXPR_MUL_1MINUS_1PLUS = 2   /* a * (1 - b) * (1 + c)  e.g. ... * (1 + l_tax) */
} gsql_expr_kind;
typedef struct gsql_derived_col {
    int32_t kind; /* gsql_expr_kind */
    int32_t a, b, c;
} gsql_derived_col;
typedef enum gsql_cmp_op { GSQL_CMP_NONE = 0, GSQL_CMP_LE = 1, GSQL_CMP_LT = 2, GSQL_CMP_GE = 3, GSQL_CMP_GT = 4, GSQL_CMP_EQ = 5, GSQL_CMP_NE = 6 } gsql_cmp_op;
#define GSQL_MAX_DERIVED 4

typedef struct gsql_agg_spec {
    int32_t n_input_cols;
    int32_t input_types[GSQL_MAX_COLS];
    int32_t ngroups;
    int32_t groups[GSQL_MAX_KEYS];
    int32_t naggs;
    gsql_agg_call aggs[GSQL_MAX_AGGS];
    int64_t expected_groups; /* planner estimate; only sizes the first table */
    int32_t n_derived;
    gsql_derived_col derived[GSQL_MAX_DERIVED];
    /* row filter `input[row_filter_col] <op> row_filter_value` on an INT/BIGINT column; rows that fail (or are NULL
     * there) are not aggregated.  GSQL_CMP_NONE = no filter. */
    int32_t row_filter_col;
    int32_t row_filter_op; /* gsql_cmp_op */
    int64_t row_filter_value;
} gsql_agg_spec;

gsql_status gsql_agg_create(gsql_ctx *ctx, const gsql_agg_spec *spec, gsql_agg **out);
gsql_status gsql_agg_consume(gsql_agg *a, const gsql_batch *batch);          /* consumeChunk */
gsql_status gsql_agg_finish(gsql_agg *a, int64_t *ngroups);                  /* buildConsume */
gsql_status gsql_agg_output_schema(gsql_agg *a, int32_t *ncols, int32_t *types /* GSQL_MAX_COLS */);
/* nextChunk: copies up to max_rows result rows (group keys || aggregate values) starting at the internal cursor
 * into `out` (out->mem says where); *out_rows == 0 means exhausted.  Every out column needs a nulls buffer. */
gsql_status gsql_agg_next(gsql_agg *a, gsql_batch *out, int64_t max_rows, int64_t *out_rows);
void gsql_agg_destroy(gsql_agg *a);

/* ------------------------------------------------------------------------------------------------ grouping sets */
/* A HashAgg over an Expand (GROUP BY ROLLUP / CUBE / GROUPING SETS, and the DISTINCT rewrites), without materialising the
 * Expand's copies.  GroupingSetsToExpandRule.java:255-300 (polardbx-optimizer core/planner/rule/) plans all of them as an
 * Expand that writes every input row once per grouping set — the group columns outside that set NULL, a BIGINT literal
 * `$e` naming the set — under a HashAgg grouping by (all keys..., $e).  The result here is exactly gsql_agg over the output
 * of EX/operator/ExpandExec.java:48-69 (every input chunk becomes one chunk per projection, in order):
 *   projections: proj[s][c] is projection s's output column c: GSQL_EXPAND_INPUT (input column `col`, its own type),
 *                GSQL_EXPAND_NULL, or GSQL_EXPAND_CONST (`value`, into an INT32 / INT64 output column).
 *   groups:      set s emits one row per distinct tuple of the group columns it references, among the rows consumed; the
 *                other group columns are written as its NULL or constant.  A set emits no row when no row was consumed
 *                (the stock aggregation is keyed, by $e at least, so even a grand total gives zero rows then).
 *   aggregates:  gsql_agg's kinds, types, NULL and FILTER rules and rounding contract; the output schema is
 *                gsql_agg_output_schema's over the Expand's output (n_output_cols == the agg spec's n_input_cols).
 *   order:       sets in Expand order; rows within a set unspecified.
 * Each root set (one no other set contains) aggregates the input through gsql_agg's kernels; every other set is merged
 * from the finished groups of the smallest finer set that contains it (k_agg_derive), so the input is read once per root.
 * Refused with GSQL_E_UNSUPPORTED (the planner keeps the stock ExpandExec + HashAggExec): FIRST_VALUE, AVG_MERGE,
 * n_derived != 0, a row filter; an aggregate argument or FILTER column that is not a reference to the same input column in
 * every set; a reference whose input type differs from the Expand output column's type; a constant in an FP64 column; no
 * group column holding pairwise distinct constants in all sets (without one, groups of different sets could coincide);
 * nsets outside 1..GSQL_MAX_SETS; whatever gsql_agg_create refuses.  Sizes, sources or columns out of range, an INT32
 * constant beyond 32 bits: GSQL_E_INVALID. */
#define GSQL_MAX_SETS 16 /* CUBE of four keys */
typedef enum gsql_expand_src { GSQL_EXPAND_INPUT = 0, GSQL_EXPAND_NULL = 1, GSQL_EXPAND_CONST = 2 } gsql_expand_src;
typedef struct gsql_expand_item {
    int32_t src; /* gsql_expand_src */
    int32_t col; /* GSQL_EXPAND_INPUT: input column */
    int64_t value; /* GSQL_EXPAND_CONST */
} gsql_expand_item;
typedef struct gsql_expand_spec {
    int32_t n_input_cols; /* the Expand's input = the batches consumed */
    int32_t input_types[GSQL_MAX_COLS];
    int32_t nsets, n_output_cols;
    gsql_expand_item proj[GSQL_MAX_SETS][GSQL_MAX_COLS];
} gsql_expand_spec;
typedef struct gsql_gsagg gsql_gsagg;
gsql_status gsql_gsagg_create(gsql_ctx *ctx, const gsql_expand_spec *expand, const gsql_agg_spec *agg /* over the Expand output */,
                              gsql_gsagg **out);
/* consumeChunk of the Expand's input (host or device; nothing referenced after return). */
gsql_status gsql_gsagg_consume(gsql_gsagg *g, const gsql_batch *batch);
/* buildConsume: finishes every set; *ngroups = the rows next() will return, all sets together. */
gsql_status gsql_gsagg_finish(gsql_gsagg *g, int64_t *ngroups);
gsql_status gsql_gsagg_output_schema(gsql_gsagg *g, int32_t *ncols, int32_t *types /* GSQL_MAX_COLS */);
/* gsql_agg_next's rules, sets in Expand order. */
gsql_status gsql_gsagg_next(gsql_gsagg *g, gsql_batch *out, int64_t max_rows, int64_t *out_rows);
void gsql_gsagg_destroy(gsql_gsagg *g);

/* ------------------------------------------------------------------------------------------------ sorted agg */
/* SortAggExec (operator/SortAggExec.java:72-135): one output row per maximal run of adjacent input rows whose group keys
 * compare equal under NumberType.compare — two NULLs are equal, NULL differs from every value, INT / BIGINT by value, DOUBLE
 * by Double.compare (-0.0 and +0.0 are different groups, every NaN equals every NaN).  Input ordered by gsql_sort or
 * gsql_merge on the group keys (any ASC / DESC mix) therefore has every group contiguous; unsorted input is not an error
 * (keys 1 1 2 1 give three rows).  Rows come out in input order of the groups' first rows; the key written is the first
 * row's, bit for bit (a NaN keeps its payload).  Output schema: gsql_agg_output_schema's.  No group keys: the whole input
 * is one group; empty input gives zero rows, with or without keys.  Floating SUM / AVG may add in any order (gsql_agg's
 * rounding contract).  FIRST_VALUE is the group's first non-NULL value in input order, NULL if all are NULL — unlike
 * gsql_agg's first-row rule, on purpose (see GSQL_AGG_FIRST_VALUE).
 * spec: a gsql_agg_spec; n_derived != 0, row_filter_op != GSQL_CMP_NONE or any filter_arg >= 0: GSQL_E_UNSUPPORTED (the
 * stock operator ignores FILTER clauses, so the planner must keep it for them); expected_groups is ignored; key and value
 * types INT32 / INT64 / FP64; naggs may be 0 (DISTINCT). */
typedef struct gsql_sortagg gsql_sortagg;
gsql_status gsql_sortagg_create(gsql_ctx *ctx, const gsql_agg_spec *spec, gsql_sortagg **out);
/* Aggregates `batch` (host or device; nothing referenced after return), continuing the group left open by the previous
 * batch.  *ready (may be NULL) = groups complete and not yet returned: all but the still-open last group.  Device memory
 * held between calls is O(groups not yet returned) plus the open group's key and states. */
gsql_status gsql_sortagg_consume(gsql_sortagg *s, const gsql_batch *batch, int64_t *ready);
/* End of input: closes the open group (if any); *ready as above.  consume after finish: GSQL_E_STATE. */
gsql_status gsql_sortagg_finish(gsql_sortagg *s, int64_t *ready);
gsql_status gsql_sortagg_output_schema(gsql_sortagg *s, int32_t *ncols, int32_t *types /* GSQL_MAX_COLS */);
/* gsql_agg_next's rules over the ready groups, in input order; may be interleaved with consume.  Every out column needs a
 * nulls buffer (else GSQL_E_INVALID and the cursor does not move). */
gsql_status gsql_sortagg_next(gsql_sortagg *s, gsql_batch *out, int64_t max_rows, int64_t *out_rows);
void gsql_sortagg_destroy(gsql_sortagg *s);

/* ------------------------------------------------------------------------------------------------ window */
/* NonFrameOverWindowExec (operator/NonFrameOverWindowExec.java:79-146): every call is a running value from the start of
 * the row's partition to the row itself, written to every row.  A row starts a partition when any partition column differs
 * from the previous row's under Object.equals: two NULLs are equal, NULL differs from every value, INT / BIGINT by value,
 * DOUBLE by Double.equals (-0.0 and +0.0 differ, every NaN equals every NaN).  Unordered input is not an error (partition
 * keys 1 1 2 1 give three partitions); no partition columns: the whole input is one partition.
 *   ROW_NUMBER  the row's 1-based position in its partition.
 *   RANK        the partition's row count at the first row of the current peer run, where peers are adjacent rows whose
 *               `cols` compare equal under Objects.equals; DENSE_RANK the number of peer runs so far.  No columns: 1.
 *   aggregates  COUNT(*), COUNT(cols), SUM (FP64 -> FP64, INT32 / INT64 -> DEC128), SUM0(INT64), AVG(FP64), MIN, MAX:
 *               gsql_agg's types and NULL rules, taken after each row.  Floating SUM / AVG may add in any order
 *               (gsql_agg's rounding contract; an all -0.0 prefix sums to +0.0).
 * reset_each_row != 0 (a ROWS CURRENT ROW .. CURRENT ROW frame): every call restarts at every row, so ROW_NUMBER / RANK /
 * DENSE_RANK are 1 and an aggregate covers the row alone.
 * Refused with GSQL_E_UNSUPPORTED (the planner keeps the stock operator): any filter_arg >= 0 (the stock operator ignores
 * FILTER), FIRST_VALUE, AVG_MERGE, other kinds, AVG over integers, SUM0 over non-BIGINT, RANK / DENSE_RANK with more than
 * 4 columns, DEC128 input columns.  Sizes or columns out of range: GSQL_E_INVALID. */
typedef struct gsql_window_spec {
    int32_t n_input_cols;
    int32_t input_types[GSQL_MAX_COLS];
    int32_t npart;                    /* 0..GSQL_MAX_KEYS */
    int32_t part_cols[GSQL_MAX_KEYS];
    int32_t ncalls;                   /* 1..GSQL_MAX_AGGS */
    gsql_agg_call calls[GSQL_MAX_AGGS];
    int32_t reset_each_row;
} gsql_window_spec;
typedef struct gsql_window gsql_window;
gsql_status gsql_window_create(gsql_ctx *ctx, const gsql_window_spec *spec, gsql_window **out);
/* The operator's output schema: the input columns, then one column per call (*ncols = n_input_cols + ncalls). */
gsql_status gsql_window_output_schema(gsql_window *w, int32_t *ncols, int32_t *types /* GSQL_MAX_COLS + GSQL_MAX_AGGS */);
/* One batch (host or device; nothing referenced after return), continuing the previous batch's last partition, peer run
 * and running values.  `out` holds the call columns only (out->ncols == ncalls, the schema's trailing types), host or
 * device, with room for in->rows rows; the input columns pass through unchanged and are not copied.  Every out column
 * needs a nulls buffer; a device out column must be aligned to its element (8 bytes for DEC128), else GSQL_E_INVALID.
 * Device input columns need no alignment.  out->rows = in->rows.  A batch of more than 2^40 rows is GSQL_E_CAPACITY. */
gsql_status gsql_window_apply(gsql_window *w, const gsql_batch *in, gsql_batch *out);
void gsql_window_destroy(gsql_window *w);

/* ------------------------------------------------------------------------------------------------ filter / project */
/* Vectorised Filter + Project in one pass (replaces operator/VectorizedFilterExec.java and
 * operator/VectorizedProjectExec.java:40-143 with the expression trees of the executor.vectorized package): rows for which the
 * filter is TRUE (NULL and FALSE drop, as VectorizedFilterExec keeps only selected positions) are compacted and every
 * output column is an expression over the input columns.  Expressions are postfix programs over a small typed stack:
 * integers are 64-bit two's complement (Java long arithmetic), doubles IEEE; any NULL operand makes arithmetic and
 * comparisons NULL; AND / OR / NOT follow SQL three-valued logic; comparisons and logic yield BIGINT 0 / 1.  Mixed
 * integer / double operands widen the integer to double.  GSQL_OP_DIV is NULL where the divisor (as a double) is zero, as
 * the reference's Divide expressions, so it needs a nullable output even over NULL-free input.
 * A program that is a single GSQL_OP_COL passes the column through with its own type. */
typedef enum gsql_expr_op {
    GSQL_OP_COL = 1,       /* push input column `arg` */
    GSQL_OP_CONST_I64 = 2, /* push k.i */
    GSQL_OP_CONST_F64 = 3, /* push k.d */
    GSQL_OP_ADD = 4, GSQL_OP_SUB = 5, GSQL_OP_MUL = 6, GSQL_OP_DIV = 7 /* always DOUBLE; NULL on a zero divisor */, GSQL_OP_NEG = 8,
    GSQL_OP_LT = 9, GSQL_OP_LE = 10, GSQL_OP_GT = 11, GSQL_OP_GE = 12, GSQL_OP_EQ = 13, GSQL_OP_NE = 14,
    GSQL_OP_AND = 15, GSQL_OP_OR = 16, GSQL_OP_NOT = 17, GSQL_OP_IS_NULL = 18,
    GSQL_OP_CAST_F64 = 19, GSQL_OP_CAST_I64 = 20 /* of a double: (long) Math.rint(d) as CastToSigned: half to even, saturating, NaN -> 0 */
} gsql_expr_op;
typedef struct gsql_expr_ins {
    int32_t op;  /* gsql_expr_op */
    int32_t arg; /* column index for GSQL_OP_COL */
    union { int64_t i; double d; } k;
} gsql_expr_ins;
#define GSQL_MAX_EXPR_INS 24
#define GSQL_MAX_EXPR_STACK 4 /* operand stack depth: held in registers */
#define GSQL_MAX_SCAN_OUT 16
typedef struct gsql_expr {
    int32_t n;
    int32_t reserved;
    gsql_expr_ins ins[GSQL_MAX_EXPR_INS];
} gsql_expr;
typedef struct gsql_scan_spec {
    int32_t n_input_cols;
    int32_t input_types[GSQL_MAX_COLS];
    int32_t has_filter;
    gsql_expr filter;
    int32_t n_out;
    int32_t reserved;
    gsql_expr out[GSQL_MAX_SCAN_OUT];
} gsql_scan_spec;
typedef struct gsql_scan gsql_scan;
gsql_status gsql_scan_create(gsql_ctx *ctx, const gsql_scan_spec *spec, gsql_scan **out);
gsql_status gsql_scan_output_schema(gsql_scan *s, int32_t *ncols, int32_t *types /* GSQL_MAX_SCAN_OUT */);
/* nextChunk over one input batch: `out` (same mem as `in`) receives the surviving rows, at most out_capacity
 * (GSQL_E_CAPACITY with *out_rows = in->rows otherwise: size it for the input).  An output column without a nulls
 * buffer must not receive a NULL (GSQL_E_INVALID).  The survivors of one 1024-row input tile are contiguous in the output and
 * in input order; the order of the tiles is unspecified. */
gsql_status gsql_scan_apply(gsql_scan *s, const gsql_batch *in, gsql_batch *out, int64_t out_capacity, int64_t *out_rows);
void gsql_scan_destroy(gsql_scan *s);

/* ------------------------------------------------------------------------------------------------ exchange */
typedef enum gsql_xchg_mode {
    GSQL_XCHG_HASH = 0,      /* PartitioningExchanger / HashPartitionFunction: ExecUtils.partition(Chunk.hashCode(channels)) */
    GSQL_XCHG_BROADCAST = 1, /* BroadcastExchanger / distribution=broadcast: every destination receives every row (push only;
                                local consumers of one GPU simply share the device batch) */
    GSQL_XCHG_RANDOM = 2     /* RandomExchanger.java:39-60: load balancing only — here round-robin by row index */
} gsql_xchg_mode;

typedef struct gsql_xchg_spec {
    int32_t n_cols;
    int32_t types[GSQL_MAX_COLS];
    int32_t n_channels;                 /* partition channels (hash keys) */
    int32_t channels[GSQL_MAX_KEYS];
    int32_t key_types[GSQL_MAX_KEYS];   /* keyTargetTypes; same as column type when no conversion */
    int32_t nparts;                     /* consumers (local exchange) or ranks (remote shuffle) */
    int32_t mode;                       /* gsql_xchg_mode */
} gsql_xchg_spec;

gsql_status gsql_xchg_create(gsql_ctx *ctx, const gsql_xchg_spec *spec, gsql_xchg **out);
/* Local hash-partition exchange: rows of `in` are grouped by destination into `out` (same schema, capacity >=
 * in->rows, same mem); part_counts[p] (host memory, nparts entries) = rows routed to p; destination p's rows are
 * out rows [sum(part_counts[0..p)), +part_counts[p]).  Order inside a destination is unspecified. */
gsql_status gsql_xchg_partition(gsql_xchg *x, const gsql_batch *in, gsql_batch *out, int64_t *part_counts);

/* Multi-GPU shuffle (one process per GPU).  Rank 0 creates the id, the caller broadcasts the 128 bytes by any
 * means (torch.distributed, the MPP coordinator), every rank calls comm_init. */
gsql_status gsql_comm_unique_id(uint8_t id[128]);
gsql_status gsql_comm_init(gsql_ctx *ctx, int32_t nranks, int32_t rank, const uint8_t id[128]);
gsql_status gsql_comm_destroy(gsql_ctx *ctx);
/* Partition `in` (device) by destination rank, exchange counts, and AllToAllv the column segments over
 * NVLink/NVSwitch.  `out` (device) must hold out_capacity rows; on GSQL_E_CAPACITY *out_rows is the need.
 * recv_counts (host, nranks entries, may be NULL) = rows received from each source rank. */
gsql_status gsql_xchg_all_to_all(gsql_xchg *x, const gsql_batch *in, gsql_batch *out, int64_t out_capacity,
                                 int64_t *out_rows, int64_t *recv_counts);

/* ---- one-pass partition-and-push shuffle over NVLink peer memory (no staging buffer, no NCCL on the data path).
 * Replaces mpp/operator/PartitionedOutputCollector.java:170-196 (partitionPage: per-destination page builders) +
 * mpp/execution/buffer/PartitionedOutputBuffer.enqueue:138-175 + mpp/operator/ExchangeClient.java:372-437 (pull).
 * Every rank owns a receive buffer (device memory mapped into all peers with CUDA IPC); a push call histograms the
 * destination of every row (ExecUtils.partition, bit-exact), publishes the counts to all peers through a peer-mapped
 * control block, and then ONE kernel per slab splits the rows by destination in shared memory and writes each
 * destination's run of every column straight into that GPU's receive buffer.  The batch is cut into `nslabs` row
 * slabs; slab k can be consumed (gsql_xchg_recv_view) while slab k+1 is still on the wire, on the exchange's own
 * stream.  All three calls are collective: every rank calls them in the same order with the same nslabs. */
#define GSQL_MAX_RANKS 16
#define GSQL_MAX_SLABS 32
/* Collective.  recv_capacity_rows: rows this rank (and every other: same value everywhere) can receive per push.
 * nullable_cols: bit c set = column c travels with a NULL mask. */
gsql_status gsql_xchg_open_p2p(gsql_xchg *x, int64_t recv_capacity_rows, uint32_t nullable_cols);
/* Collective, asynchronous.  `in` is device-resident and must stay unchanged until the last slab has been waited for
 * (gsql_xchg_recv_view) or gsql_xchg_push_wait returns.  slab_rows (host, nslabs entries) = rows this rank receives in
 * each slab.  GSQL_E_CAPACITY (with *total_rows = the largest need of any rank) is returned on EVERY rank when any
 * rank's buffer would overflow — nothing is sent.  A push overwrites the rows received by the previous push. */
gsql_status gsql_xchg_push(gsql_xchg *x, const gsql_batch *in, int32_t nslabs, int64_t *slab_rows, int64_t *total_rows);
/* Makes the context stream wait for slab `slab` of the last push and describes it in place (zero copy): view->cols must
 * have n_cols entries; data/nulls point into the receive buffer, rows = slab_rows[slab].  slab = -1: all slabs as one
 * batch (they are contiguous).  The view is valid until the next push on this handle. */
gsql_status gsql_xchg_recv_view(gsql_xchg *x, int32_t slab, gsql_batch *view);
/* Blocks the host until every slab of the last push has been sent and received. */
gsql_status gsql_xchg_push_wait(gsql_xchg *x);
/* Host-side layout arithmetic of a push, exported so that it can be tested without a GPU: matrix[src][slab][dst]
 * (nranks*nslabs*nranks entries) -> send_base[slab][dst] = first row of this rank's (slab, dst) segment inside dst's
 * receive buffer, recv_base[slab][src] = first row of src's segment of that slab in this rank's buffer,
 * slab_rows[slab]; returns the largest number of rows any rank receives. */
int64_t gsql_xchg_plan_layout(int32_t nranks, int32_t nslabs, int32_t me, const int64_t *matrix, int64_t *send_base,
                              int64_t *recv_base, int64_t *slab_rows);
void gsql_xchg_destroy(gsql_xchg *x);

/* ------------------------------------------------------------------------------------------------ wire codec */
/* The MPP wire format of a Chunk (mpp/execution/buffer/PagesSerde.java:57-115 uncompressed path,
 * PagesSerdeUtil.java:36-58 writeRawPage / readRawPage, :50-58 + :60-67 the SerializedChunk framing,
 * chunk/{Integer,Long,Double}BlockEncoding.java + EncoderUtil.java:43-150), so that a GPU task can exchange pages with
 * stock Java tasks on other nodes.  All integers little-endian (airlift Slice).  A batch becomes consecutive pages of
 * `page_rows` rows:
 *     page   := int32 positionCount | int8 marker (0 = UNCOMPRESSED) | int32 uncompressedSize | int32 sizeInBytes | raw
 *     raw    := int32 blockCount | block*
 *     block  := int32 positionCount | nullbits (ceil(n/8) bytes, first row = most significant bit) | non-NULL values in row order
 * Compression (the optional LZ4 step of PagesSerde) is not produced; compressed pages are rejected by deserialize. */
/* Serialized size of `in` cut into pages of page_rows rows (exact; needs one pass over the NULL masks).  GSQL_E_UNSUPPORTED
 * when a page's payload would exceed INT32_MAX bytes (sizeInBytes is an int32). */
gsql_status gsql_serde_size(gsql_ctx *ctx, const gsql_batch *in, int32_t page_rows, int64_t *bytes);
/* `out_bytes` lives in in->mem.  GSQL_E_CAPACITY with *bytes = the need when capacity is too small; GSQL_E_UNSUPPORTED as
 * gsql_serde_size. */
gsql_status gsql_serde_serialize(gsql_ctx *ctx, const gsql_batch *in, int32_t page_rows, void *out_bytes, int64_t capacity, int64_t *bytes);
/* Decodes every page of `bytes` (host or device, `mem`) into `out` (same mem; out->ncols columns of `types`, each with a
 * nulls buffer, capacity out_capacity rows).  The bytes come from the network, so every page is checked on the host before
 * anything is decoded, as the reference reads a page from a slice bounded by its sizeInBytes: the frame must fit the
 * buffer, its marker be 0 and uncompressedSize equal sizeInBytes; blockCount must equal out->ncols; each block's
 * positionCount must equal the frame's, and its 4-byte header, its ceil(n/8)-byte NULL bit stream and one value per clear
 * bit must lie inside the page.  Bytes after a page's last block are ignored.  Any violation is GSQL_E_INVALID, reported
 * before GSQL_E_CAPACITY and with `out`'s buffers untouched; GSQL_E_CAPACITY (with *out_rows = the need) only for a
 * well-formed stream. */
gsql_status gsql_serde_deserialize(gsql_ctx *ctx, const void *bytes, int64_t nbytes, int32_t mem, gsql_batch *out, int64_t out_capacity,
                                   int64_t *out_rows);

/* ------------------------------------------------------------------------------------------------ runtime filter */
/* The bloom filter of a runtime-filtered INNER / SEMI hash join (JoinToRuntimeFilterJoinRule.java:85,172-228), bit-compatible
 * with common/utils/bloomfilter/BloomFilter.java under the xxhash_64 method (HashMethodInfo.XXHASH_METHOD): the bitmap is
 * the reference's long[numBits/64] (bit i = word[i >> 6] & (1 << (i & 63))), so a filter built here merges with filters
 * of stock Java tasks and vice versa.  One key column per filter (the planner ANDs one filter per key column).  Key
 * columns are INT32 (sign-extended), INT64 or FP64 (raw bits: -0.0 and +0.0 differ); a NULL key hashes as 0. */
typedef struct gsql_bloom gsql_bloom;
/* BloomFilter.createEmpty(method, numHashFunctions, numBits).  xxhash_64 only; num_bits % 64 == 0,
 * 64 <= num_bits <= 2^31-64 (BloomFilter.java:45 multiplyExact) and k >= 1, else GSQL_E_INVALID; k > 64: GSQL_E_UNSUPPORTED. */
gsql_status gsql_bloom_create(gsql_ctx *ctx, int64_t num_bits, int32_t num_hash_functions, gsql_bloom **out);
/* BloomFilterProduce.addChunk:92-106: puts the key column of every row (BloomFilter.put64). */
gsql_status gsql_bloom_put(gsql_bloom *b, const gsql_batch *batch, int32_t key_col);
/* BloomFilter.merge / createWithData: ORs `nfilters` bitmaps of num_bits/64 words each, stored back to back in `words`
 * (host or device, `mem`), into the filter. */
gsql_status gsql_bloom_merge(gsql_bloom *b, const uint64_t *words, int64_t nfilters, int32_t mem);
/* BloomFilter.getBitmap(): copies the num_bits/64 words into `words` (host or device, `mem`). */
gsql_status gsql_bloom_bitmap(gsql_bloom *b, uint64_t *words, int32_t mem);
/* FilterExec with condition BLOOMFILTER(key) (FilterExec.java:81-130): `out` (same mem, same columns and types as `in`)
 * receives the rows whose key mightContain64 accepts.  Capacity and NULL-buffer rules are gsql_scan_apply's. */
gsql_status gsql_bloom_filter(gsql_bloom *b, const gsql_batch *in, int32_t key_col, gsql_batch *out, int64_t out_capacity,
                              int64_t *out_rows);
void gsql_bloom_destroy(gsql_bloom *b);

/* ------------------------------------------------------------------------------------------------ sort / top-n */
/* ORDER BY (operator/SortExec.java + operator/util/MemSortor.java:60-78) and ORDER BY ... LIMIT
 * (operator/SpilledTopNExec.java:66-70).  Rows come out in the order of the executor's comparator,
 * utils/ExecUtils.getComparator:451-490: keys compare in order, two NULLs are equal and NULL is the smallest value
 * (NumberType.compare), DESC negates, so NULLs lead under ASC and trail under DESC — the collation's null direction is
 * never consulted, hence no field for it.  INT / BIGINT in natural order (a DATE arrives as a packed BIGINT and sorts as
 * one), DOUBLE by Double.compareTo (-0.0 < +0.0, every NaN equal and above +Inf).  Rows with equal keys come out in
 * unspecified order (IntArrays.quickSort is not stable), and which rows tied at a top-n boundary survive is unspecified. */
typedef struct gsql_sort_spec {
    int32_t n_cols;
    int32_t types[GSQL_MAX_COLS]; /* INT32 / INT64 / FP64; DEC128 anywhere: GSQL_E_UNSUPPORTED */
    int32_t nkeys;                /* 1..GSQL_MAX_KEYS */
    int32_t key_col[GSQL_MAX_KEYS];
    int32_t key_desc[GSQL_MAX_KEYS]; /* 0 = ASC, 1 = DESC */
    int64_t limit;                /* -1: full sort (SortExec); >= 0: top-n of topSize = skip + fetch rows; < -1: GSQL_E_INVALID */
} gsql_sort_spec;
typedef struct gsql_sort gsql_sort;
/* Each rejection names its reason in gsql_last_error. */
gsql_status gsql_sort_create(gsql_ctx *ctx, const gsql_sort_spec *spec, gsql_sort **out);
/* consumeChunk: host or device batch of the spec's columns; nothing of `batch` is referenced after return.  A full sort
 * holds every row (GSQL_E_CAPACITY past 2^31-1 rows: row ids are 32-bit; GSQL_E_OOM when HBM runs out; no spill); a top-n
 * cuts every batch to its best `limit` rows on arrival and holds O(limit) rows. */
gsql_status gsql_sort_consume(gsql_sort *s, const gsql_batch *batch);
/* buildConsume: orders what was consumed; *rows = the number of rows next() will return. */
gsql_status gsql_sort_finish(gsql_sort *s, int64_t *rows);
/* nextChunk: copies up to max_rows rows in order from the internal cursor into `out` (out->mem says where; the spec's
 * columns); *out_rows == 0 means exhausted.  An out column whose `nulls` is NULL must not receive a NULL (GSQL_E_INVALID,
 * the cursor does not move). */
gsql_status gsql_sort_next(gsql_sort *s, gsql_batch *out, int64_t max_rows, int64_t *out_rows);
void gsql_sort_destroy(gsql_sort *s);

/* ------------------------------------------------------------------------------------------------ merge of sorted runs */
/* The merge under every ORDER BY of an MPP plan: operator/MergeSortExec.java (the local drivers' runs, built by
 * LocalMergeSortExecutorFactory) and operator/SortMergeExchangeExec.java:151-160 (the remote tasks' runs) both call
 * operator/util/MergeSortedChunks.mergeSortedPages with ChunkWithPositionComparator, which is ExecUtils.getComparator.
 * `n_inputs` inputs, each already ordered under that comparator, come out as one sequence in that order:
 *   order:    exactly gsql_sort's (NULL is the smallest value, DESC negates, doubles by Double.compareTo);
 *   ties:     the merge is stable: rows with equal keys come out input by input in index order, and within an input in
 *             arrival order (the reference's priority queue leaves this unspecified; stable is stricter);
 *   unsorted: an input that is not ordered gives an unspecified output order, but every held row comes out exactly once;
 *   limit:    spec->limit = -1: every row; >= 0: the first `limit` rows (= offset + fetch: the caller skips `offset`, as
 *             GpuTopNExecutorFactory does).  An input contributes at most `limit` rows: consume drops that input's rows
 *             past its quota, so a top-n merge holds at most n_inputs * limit rows;
 *   capacity: more than 2^31-1 held rows: GSQL_E_CAPACITY (row ids are 32-bit, as in the sort).
 * Errors: n_inputs outside [1, GSQL_MAX_MERGE_INPUTS] or an input index out of range: GSQL_E_INVALID; consume after
 * finish: GSQL_E_STATE; DEC128 columns: GSQL_E_UNSUPPORTED; the spec is otherwise checked as gsql_sort_create checks it. */
#define GSQL_MAX_MERGE_INPUTS 4096
typedef struct gsql_merge gsql_merge;
gsql_status gsql_merge_create(gsql_ctx *ctx, const gsql_sort_spec *spec, int32_t n_inputs, gsql_merge **out);
/* Appends `batch` (host or device, the spec's columns) to input `input`.  Chunks of one input arrive in order; chunks of
 * different inputs may interleave.  Copies: nothing of `batch` is referenced after return. */
gsql_status gsql_merge_consume(gsql_merge *m, int32_t input, const gsql_batch *batch);
/* Merges what was consumed; *rows = the number of rows next() will return. */
gsql_status gsql_merge_finish(gsql_merge *m, int64_t *rows);
/* gsql_sort_next's rules: up to max_rows rows in order into `out`; *out_rows == 0 means exhausted. */
gsql_status gsql_merge_next(gsql_merge *m, gsql_batch *out, int64_t max_rows, int64_t *out_rows);
void gsql_merge_destroy(gsql_merge *m);

/* ------------------------------------------------------------------------------------------------ sort-merge join */
/* SortMergeJoinExec (operator/SortMergeJoinExec.java:186-278, 375-455, 547-567): joins an outer and an inner input that are
 * both ordered on the join keys, and keeps the stock operator's row order.
 *   keys:   converted to key_type (gsql_load_key's rules) and compared key by key by NumberType.compare, negated where
 *           key_desc[k] == 1: two NULLs are equal and NULL is the smallest value (the largest under DESC); INT / BIGINT by
 *           value; DOUBLE by Double.compareTo, so -0.0 and +0.0 do not join and NaN joins NaN.  A row with a NULL in any
 *           key column matches nothing.
 *   order:  outer input order.  INNER / LEFT / RIGHT: a matched outer row is followed by its run of equal-key inner rows in
 *           inner order; LEFT / RIGHT add one NULL-padded row per unmatched outer row.  SEMI: each matched outer row
 *           once.  ANTI: each unmatched outer row whose anti operands are all non-NULL, or every unmatched row when the
 *           inner side is empty.  RIGHT: the outer side is the right input; columns are inner || outer.
 *   schema: gsql_join_output_schema's rule.
 *   NOT IN: ANTI with anti operands, a non-empty inner side and a NULL in any key of the FIRST inner row produces no rows
 *           (the stock check; under DESC a NULL that is not first is not seen, on purpose).
 *   single: max_one_row with INNER / LEFT: outer columns + the first inner column; an outer row with a non-NULL key and two
 *           or more inner matches is GSQL_E_MORE_THAN_ONE_ROW at the probe of its batch.
 *   refused (GSQL_E_UNSUPPORTED, the planner keeps the stock operator): n_cond != 0, build_outer, max_one_row with SEMI /
 *           ANTI / RIGHT, DEC128 columns or keys, nkeys outside 1..GSQL_MAX_KEYS.
 *   unordered input: GSQL_E_INVALID naming the side, for inner rows out of order, outer rows out of order within a batch,
 *           or an outer batch whose first row sorts before the previous batch's last row.
 * The inner side is held whole in HBM: more than 2^31-1 inner rows is GSQL_E_CAPACITY (32-bit row ids), as is an outer
 * batch of more than 2^31-2 rows (its n + 1 output offsets are scanned with a 32-bit item count). */
typedef struct gsql_smj gsql_smj;
gsql_status gsql_smj_create(gsql_ctx *ctx, const gsql_join_spec *spec, const int32_t *key_desc /* nkeys: 0 ASC, 1 DESC */,
                            gsql_smj **out);
/* Appends (copies) an inner batch; inner batches arrive in order. */
gsql_status gsql_smj_inner_consume(gsql_smj *s, const gsql_batch *inner);
/* End of the inner input: key images, order check, run table. */
gsql_status gsql_smj_inner_finish(gsql_smj *s);
gsql_status gsql_smj_output_schema(gsql_smj *s, int32_t *ncols, int32_t *types /* GSQL_MAX_COLS*2 */);
/* Joins the next outer batch; *out_rows = the exact number of rows next() will return for it (64-bit: it may exceed
 * 2^32).  A host batch is uploaded; a device batch is referenced, not copied, and must stay valid and unchanged until
 * next() returns 0 rows.  Before inner_finish, or while rows of the previous batch are left: GSQL_E_STATE. */
gsql_status gsql_smj_probe(gsql_smj *s, const gsql_batch *outer, int64_t *out_rows);
/* gsql_sort_next's rules: the current batch's rows in order from a cursor; *out_rows == 0 means the batch is exhausted.
 * A NULL bound for a column without a nulls buffer is GSQL_E_INVALID and the cursor does not move. */
gsql_status gsql_smj_next(gsql_smj *s, gsql_batch *out, int64_t max_rows, int64_t *out_rows);
void gsql_smj_destroy(gsql_smj *s);

#if defined(__GNUC__)
#pragma GCC visibility pop
#endif
#ifdef __cplusplus
}
#endif
#endif /* GSQL_GPU_H */
