/*
 * gsql_jni.c — thin JNI shim between com.alibaba.polardbx.executor.operator.gpu.GpuNative and libgsql_gpu.so.
 *
 * Build where the CN is built:
 *   gcc -shared -fPIC -I$JAVA_HOME/include -I$JAVA_HOME/include/linux -I../include gsql_jni.c -L<dir> -lgsql_gpu -o libgsql_jni.so
 * In this repository (no JDK) tests/test_jni_boundary.py compiles and links it against jni/stub/jni.h, and checks that
 * every `native` of GpuNative.java has its Java_..._GpuNative_<name> here and vice versa.
 *
 * A "staging" object is a set of pinned host column buffers (gsql_host_alloc) that Java fills chunk by chunk with
 * GetPrimitiveArrayCritical + memcpy ("pins Chunk blocks into device memory" = array -> pinned -> cudaMemcpyAsync inside
 * the library).  It tracks per column whether any appended row was NULL and passes `nulls = NULL` to the library
 * otherwise — AbstractBlock.mayHaveNull() == false — so that NULL-free inputs take the packed-row fast paths (the
 * library additionally drops all-zero masks on its own).  Non-zero gsql_status becomes GpuExecutorException
 * (TddlRuntimeException / ERR_EXECUTOR, message = gsql_last_error) — or GpuMoreThanOneRowException for
 * GSQL_E_MORE_THAN_ONE_ROW (ERR_SCALAR_SUBQUERY_RETURN_MORE_THAN_ONE_ROW, AbstractBufferedJoinExec.java:217-219).
 */
#include <jni.h>
#include <stdlib.h>
#include <string.h>

#include "gsql_gpu.h"

#define NATIVE(ret, name) JNIEXPORT ret JNICALL Java_com_alibaba_polardbx_executor_operator_gpu_GpuNative_##name

typedef struct staging {
    int32_t ncols;
    int32_t types[GSQL_MAX_COLS * 2];
    int64_t cap, rows;
    void *data[GSQL_MAX_COLS * 2];
    uint8_t *nulls[GSQL_MAX_COLS * 2];
    int any_null[GSQL_MAX_COLS * 2]; /* some appended row of this column was NULL */
    int outputs;                      /* used as an output batch: every column hands a mask to the library */
    gsql_col cols[GSQL_MAX_COLS * 2];
    gsql_batch batch;
} staging;

/* every handle remembers its context so that errors can carry gsql_last_error */
typedef struct jhandle {
    gsql_ctx *ctx;
    void *h;
} jhandle;

static int width(int t) { return t == GSQL_T_INT32 ? 4 : t == GSQL_T_DEC128 ? 16 : 8; }

static void throw_status(JNIEnv *env, gsql_ctx *ctx, int st) {
    const char *cls = st == GSQL_E_MORE_THAN_ONE_ROW ? "com/alibaba/polardbx/executor/operator/gpu/GpuMoreThanOneRowException"
                                                     : "com/alibaba/polardbx/executor/operator/gpu/GpuExecutorException";
    if ((*env)->ExceptionCheck(env)) return;
    (*env)->ThrowNew(env, (*env)->FindClass(env, cls), ctx ? gsql_last_error(ctx) : "gsql error (no context)");
}

/* input view: a column without any NULL so far goes in as nulls = NULL */
static gsql_batch *as_batch(staging *s, int output) {
    for (int i = 0; i < s->ncols; i++) {
        s->cols[i].type = s->types[i];
        s->cols[i].reserved = 0;
        s->cols[i].data = s->data[i];
        s->cols[i].nulls = (output || s->any_null[i]) ? s->nulls[i] : NULL;
    }
    s->batch.rows = output ? 0 : s->rows;
    s->batch.ncols = s->ncols;
    s->batch.mem = GSQL_MEM_HOST;
    s->batch.cols = s->cols;
    return &s->batch;
}

static int staging_reserve(staging *s, int64_t rows) {
    if (rows <= s->cap) return 0;
    int64_t cap = s->cap ? s->cap : 4096;
    while (cap < rows) cap *= 2;
    for (int i = 0; i < s->ncols; i++) {
        void *nd = NULL, *nn = NULL;
        if (gsql_host_alloc((size_t)cap * width(s->types[i]), &nd) != GSQL_OK) return -1;
        if (gsql_host_alloc((size_t)cap, &nn) != GSQL_OK) { gsql_host_free(nd); return -1; }
        if (s->rows) {
            memcpy(nd, s->data[i], (size_t)s->rows * width(s->types[i]));
            memcpy(nn, s->nulls[i], (size_t)s->rows);
        }
        gsql_host_free(s->data[i]);
        gsql_host_free(s->nulls[i]);
        s->data[i] = nd;
        s->nulls[i] = (uint8_t *)nn;
    }
    s->cap = cap;
    return 0;
}

/* an output batch has just been filled by the library: recompute the per-column NULL summary for `rows` rows */
static void staging_filled(staging *s, int64_t rows) {
    s->rows = rows;
    for (int i = 0; i < s->ncols; i++) {
        int any = 0;
        const uint8_t *m = s->nulls[i];
        for (int64_t r = 0; r < rows && !any; r++) any = m[r] != 0;
        s->any_null[i] = any;
    }
}

static void fill_ints(JNIEnv *env, jintArray a, int32_t *dst, int32_t *n, int max) {
    *n = a ? (*env)->GetArrayLength(env, a) : 0;
    if (*n > max) *n = max;
    if (*n) (*env)->GetIntArrayRegion(env, a, 0, *n, (jint *)dst);
}

/* ---- context ------------------------------------------------------------------------------------------------ */
NATIVE(jlong, ctxCreate)(JNIEnv *env, jclass c, jint device) {
    gsql_ctx *ctx = NULL;
    int st = gsql_ctx_create(device, &ctx);
    if (st != GSQL_OK) throw_status(env, NULL, st); /* no CPU fallback: the planner must not have chosen this operator */
    return (jlong)(intptr_t)ctx;
}

NATIVE(void, ctxDestroy)(JNIEnv *env, jclass c, jlong ctx) { gsql_ctx_destroy((gsql_ctx *)(intptr_t)ctx); }

NATIVE(jint, deviceCount)(JNIEnv *env, jclass c) {
    int n = 0;
    for (;; n++) { /* the ABI has no device-count call: probe contexts until one fails */
        gsql_ctx *ctx = NULL;
        if (n >= 64 || gsql_ctx_create(n, &ctx) != GSQL_OK) break;
        gsql_ctx_destroy(ctx);
    }
    return n;
}

/* ---- staging ------------------------------------------------------------------------------------------------ */
NATIVE(jlong, stagingCreate)(JNIEnv *env, jclass c, jintArray types, jint cap) {
    staging *s = (staging *)calloc(1, sizeof(staging));
    if (!s) return 0;
    fill_ints(env, types, s->types, &s->ncols, GSQL_MAX_COLS * 2);
    if (staging_reserve(s, cap > 0 ? cap : 1)) throw_status(env, NULL, GSQL_E_OOM);
    return (jlong)(intptr_t)s;
}

/* Block arrays -> pinned staging.  columns[i] is int[] / long[] / double[] (IntegerBlock.intArray():217,
 * LongBlock.longArray():191, DoubleBlock.doubleArray():190), nulls[i] is boolean[] or null (AbstractBlock.nulls():116).
 * sel == NULL: rows [offset, offset+rows) of every array; else row i is element sel[i] (Chunk.selection()). */
static void append_rows(JNIEnv *env, staging *s, jobjectArray columns, jobjectArray nulls, jint offset, const jint *sel, jint rows) {
    if (staging_reserve(s, s->rows + rows)) { throw_status(env, NULL, GSQL_E_OOM); return; }
    for (int i = 0; i < s->ncols; i++) {
        const int w = width(s->types[i]);
        jarray col = (jarray)(*env)->GetObjectArrayElement(env, columns, i);
        jarray nl = nulls ? (jarray)(*env)->GetObjectArrayElement(env, nulls, i) : NULL;
        char *dst = (char *)s->data[i] + (size_t)s->rows * w;
        uint8_t *dn = s->nulls[i] + s->rows;
        void *p = (*env)->GetPrimitiveArrayCritical(env, col, NULL);
        if (!sel) {
            memcpy(dst, (char *)p + (size_t)offset * w, (size_t)rows * w);
        } else if (w == 4) {
            for (jint r = 0; r < rows; r++) ((int32_t *)dst)[r] = ((const int32_t *)p)[sel[r]];
        } else {
            for (jint r = 0; r < rows; r++) ((int64_t *)dst)[r] = ((const int64_t *)p)[sel[r]];
        }
        (*env)->ReleasePrimitiveArrayCritical(env, col, p, JNI_ABORT);
        if (nl) {
            const uint8_t *q = (const uint8_t *)(*env)->GetPrimitiveArrayCritical(env, nl, NULL); /* jboolean is one byte */
            int any = 0;
            if (!sel) {
                memcpy(dn, q + offset, (size_t)rows);
                for (jint r = 0; r < rows; r++) any |= dn[r];
            } else {
                for (jint r = 0; r < rows; r++) { dn[r] = q[sel[r]]; any |= dn[r]; }
            }
            (*env)->ReleasePrimitiveArrayCritical(env, nl, (void *)q, JNI_ABORT);
            if (any) s->any_null[i] = 1;
            (*env)->DeleteLocalRef(env, nl);
        } else {
            memset(dn, 0, (size_t)rows);
        }
        (*env)->DeleteLocalRef(env, col);
    }
    s->rows += rows;
}

NATIVE(void, stagingAppend)(JNIEnv *env, jclass c, jlong h, jobjectArray columns, jobjectArray nulls, jint offset, jint rows) {
    append_rows(env, (staging *)(intptr_t)h, columns, nulls, offset, NULL, rows);
}

NATIVE(void, stagingAppendSelected)(JNIEnv *env, jclass c, jlong h, jobjectArray columns, jobjectArray nulls, jintArray selection, jint rows) {
    jint *sel = (jint *)malloc((size_t)(rows > 0 ? rows : 1) * sizeof(jint));
    if (!sel) { throw_status(env, NULL, GSQL_E_OOM); return; }
    (*env)->GetIntArrayRegion(env, selection, 0, rows, sel);
    append_rows(env, (staging *)(intptr_t)h, columns, nulls, 0, sel, rows);
    free(sel);
}

NATIVE(jint, stagingRows)(JNIEnv *env, jclass c, jlong h) { return (jint)((staging *)(intptr_t)h)->rows; }

NATIVE(void, stagingReset)(JNIEnv *env, jclass c, jlong h) {
    staging *s = (staging *)(intptr_t)h;
    s->rows = 0;
    memset(s->any_null, 0, sizeof(s->any_null));
}

NATIVE(void, stagingDestroy)(JNIEnv *env, jclass c, jlong h) {
    staging *s = (staging *)(intptr_t)h;
    if (!s) return;
    for (int i = 0; i < s->ncols; i++) {
        gsql_host_free(s->data[i]);
        gsql_host_free(s->nulls[i]);
    }
    free(s);
}

NATIVE(jobject, stagingColumn)(JNIEnv *env, jclass c, jlong h, jint col, jint from, jint rows) {
    staging *s = (staging *)(intptr_t)h;
    if (col < 0 || col >= s->ncols || from < 0 || rows < 0 || (int64_t)from + rows > s->rows) { throw_status(env, NULL, GSQL_E_INVALID); return NULL; }
    switch (s->types[col]) {
    case GSQL_T_INT32: {
        jintArray a = (*env)->NewIntArray(env, rows);
        if (a) (*env)->SetIntArrayRegion(env, a, 0, rows, (const jint *)s->data[col] + from);
        return a;
    }
    case GSQL_T_FP64: {
        jdoubleArray a = (*env)->NewDoubleArray(env, rows);
        if (a) (*env)->SetDoubleArrayRegion(env, a, 0, rows, (const jdouble *)s->data[col] + from);
        return a;
    }
    case GSQL_T_DEC128: { /* two longs per row: lo, hi */
        jlongArray a = (*env)->NewLongArray(env, rows * 2);
        if (a) (*env)->SetLongArrayRegion(env, a, 0, rows * 2, (const jlong *)s->data[col] + (size_t)from * 2);
        return a;
    }
    default: {
        jlongArray a = (*env)->NewLongArray(env, rows);
        if (a) (*env)->SetLongArrayRegion(env, a, 0, rows, (const jlong *)s->data[col] + from);
        return a;
    }
    }
}

NATIVE(jbooleanArray, stagingNulls)(JNIEnv *env, jclass c, jlong h, jint col, jint from, jint rows) {
    staging *s = (staging *)(intptr_t)h;
    if (col < 0 || col >= s->ncols || from < 0 || rows < 0 || (int64_t)from + rows > s->rows) { throw_status(env, NULL, GSQL_E_INVALID); return NULL; }
    if (!s->any_null[col]) return NULL;
    const uint8_t *m = s->nulls[col] + from;
    int any = 0;
    for (jint r = 0; r < rows && !any; r++) any = m[r] != 0;
    if (!any) return NULL;
    jbooleanArray a = (*env)->NewBooleanArray(env, rows);
    if (a) (*env)->SetBooleanArrayRegion(env, a, 0, rows, (const jboolean *)m);
    return a;
}

/* ---- join --------------------------------------------------------------------------------------------------- */
NATIVE(jlong, joinCreate)(JNIEnv *env, jclass c, jlong ctx, jint joinType, jboolean maxOneRow, jboolean buildOuter, jintArray outerKeys,
                          jintArray innerKeys, jintArray keyTypes, jintArray outerTypes, jintArray innerTypes, jintArray antiOperands,
                          jintArray condCols, jlongArray condNe, jlong expectedBuildRows) {
    gsql_join_spec s;
    memset(&s, 0, sizeof(s));
    int32_t n;
    s.join_type = joinType;
    s.max_one_row = maxOneRow;
    s.build_outer = buildOuter;
    fill_ints(env, outerKeys, s.outer_key, &s.nkeys, GSQL_MAX_KEYS);
    fill_ints(env, innerKeys, s.inner_key, &n, GSQL_MAX_KEYS);
    fill_ints(env, keyTypes, s.key_type, &n, GSQL_MAX_KEYS);
    fill_ints(env, outerTypes, s.outer_types, &s.n_outer_cols, GSQL_MAX_COLS);
    fill_ints(env, innerTypes, s.inner_types, &s.n_inner_cols, GSQL_MAX_COLS);
    fill_ints(env, antiOperands, s.anti_operands, &s.n_anti_operands, GSQL_MAX_KEYS);
    fill_ints(env, condCols, s.cond_col, &s.n_cond, 4);
    if (s.n_cond) (*env)->GetLongArrayRegion(env, condNe, 0, s.n_cond, (jlong *)s.cond_ne_value);
    s.expected_build_rows = expectedBuildRows;
    gsql_join *j = NULL;
    int st = gsql_join_create((gsql_ctx *)(intptr_t)ctx, &s, &j);
    if (st != GSQL_OK) { throw_status(env, (gsql_ctx *)(intptr_t)ctx, st); return 0; }
    jhandle *h = (jhandle *)calloc(1, sizeof(jhandle));
    h->ctx = (gsql_ctx *)(intptr_t)ctx;
    h->h = j;
    return (jlong)(intptr_t)h;
}

NATIVE(void, joinBuildConsume)(JNIEnv *env, jclass c, jlong jh, jlong sh) {
    jhandle *h = (jhandle *)(intptr_t)jh;
    int st = gsql_join_build_consume((gsql_join *)h->h, as_batch((staging *)(intptr_t)sh, 0));
    if (st != GSQL_OK) throw_status(env, h->ctx, st);
}

NATIVE(void, joinBuildFinish)(JNIEnv *env, jclass c, jlong jh) {
    jhandle *h = (jhandle *)(intptr_t)jh;
    int st = gsql_join_build_finish((gsql_join *)h->h);
    if (st != GSQL_OK) throw_status(env, h->ctx, st);
}

NATIVE(jint, joinProbe)(JNIEnv *env, jclass c, jlong jh, jlong ph, jlong oh) {
    jhandle *h = (jhandle *)(intptr_t)jh;
    staging *p = (staging *)(intptr_t)ph, *o = (staging *)(intptr_t)oh;
    int64_t rows = 0;
    if (staging_reserve(o, p->rows)) { throw_status(env, NULL, GSQL_E_OOM); return -1; } /* <= 1 row per probe row keeps the fast path */
    for (;;) {
        int st = gsql_join_probe((gsql_join *)h->h, as_batch(p, 0), as_batch(o, 1), o->cap, &rows);
        if (st == GSQL_E_CAPACITY) { /* duplicate build keys: the library tells the exact need */
            if (staging_reserve(o, rows)) { throw_status(env, NULL, GSQL_E_OOM); return -1; }
            continue;
        }
        if (st != GSQL_OK) { throw_status(env, h->ctx, st); return -1; }
        staging_filled(o, rows);
        return (jint)rows;
    }
}

NATIVE(jint, joinUnmatchedBuild)(JNIEnv *env, jclass c, jlong jh, jlong oh) {
    jhandle *h = (jhandle *)(intptr_t)jh;
    staging *o = (staging *)(intptr_t)oh;
    int64_t rows = 0;
    for (;;) {
        int st = gsql_join_unmatched_build((gsql_join *)h->h, as_batch(o, 1), o->cap, &rows);
        if (st == GSQL_E_CAPACITY) {
            if (staging_reserve(o, rows)) { throw_status(env, NULL, GSQL_E_OOM); return -1; }
            continue;
        }
        if (st != GSQL_OK) { throw_status(env, h->ctx, st); return -1; }
        staging_filled(o, rows);
        return (jint)rows;
    }
}

NATIVE(jlong, joinDeviceBytes)(JNIEnv *env, jclass c, jlong jh) {
    jhandle *h = (jhandle *)(intptr_t)jh;
    gsql_join_info info;
    if (gsql_join_info_get((gsql_join *)h->h, &info) != GSQL_OK) return 0;
    return (jlong)info.device_bytes;
}

NATIVE(void, joinDestroy)(JNIEnv *env, jclass c, jlong jh) {
    jhandle *h = (jhandle *)(intptr_t)jh;
    if (!h) return;
    gsql_join_destroy((gsql_join *)h->h);
    free(h);
}

/* ---- aggregation -------------------------------------------------------------------------------------------- */
static int fill_agg_spec(JNIEnv *env, gsql_agg_spec *s, jintArray inputTypes, jintArray groups, jintArray aggKinds, jobjectArray aggCols,
                         jintArray filterArgs, jlong expectedGroups) {
    memset(s, 0, sizeof(*s));
    int32_t kinds[GSQL_MAX_AGGS], fargs[GSQL_MAX_AGGS], n;
    fill_ints(env, inputTypes, s->input_types, &s->n_input_cols, GSQL_MAX_COLS);
    fill_ints(env, groups, s->groups, &s->ngroups, GSQL_MAX_KEYS);
    fill_ints(env, aggKinds, kinds, &s->naggs, GSQL_MAX_AGGS);
    fill_ints(env, filterArgs, fargs, &n, GSQL_MAX_AGGS);
    for (int i = 0; i < s->naggs; i++) {
        jintArray cols = aggCols ? (jintArray)(*env)->GetObjectArrayElement(env, aggCols, i) : NULL;
        s->aggs[i].kind = kinds[i];
        s->aggs[i].filter_arg = i < n ? fargs[i] : -1;
        fill_ints(env, cols, s->aggs[i].cols, &s->aggs[i].ncols, 4);
        if (cols) (*env)->DeleteLocalRef(env, cols);
    }
    s->expected_groups = expectedGroups;
    s->row_filter_col = -1;
    s->row_filter_op = GSQL_CMP_NONE;
    return 0;
}

static jlong agg_create(JNIEnv *env, jlong ctx, const gsql_agg_spec *s) {
    gsql_agg *a = NULL;
    int st = gsql_agg_create((gsql_ctx *)(intptr_t)ctx, s, &a);
    if (st != GSQL_OK) { throw_status(env, (gsql_ctx *)(intptr_t)ctx, st); return 0; }
    jhandle *h = (jhandle *)calloc(1, sizeof(jhandle));
    h->ctx = (gsql_ctx *)(intptr_t)ctx;
    h->h = a;
    return (jlong)(intptr_t)h;
}

NATIVE(jlong, aggCreate)(JNIEnv *env, jclass c, jlong ctx, jintArray inputTypes, jintArray groups, jintArray aggKinds, jobjectArray aggCols,
                         jintArray filterArgs, jlong expectedGroups) {
    gsql_agg_spec s;
    fill_agg_spec(env, &s, inputTypes, groups, aggKinds, aggCols, filterArgs, expectedGroups);
    return agg_create(env, ctx, &s);
}

/* aggregation with the Project / Filter under it fused in (gsql_agg_spec.derived / row_filter_*) */
NATIVE(jlong, aggCreateFused)(JNIEnv *env, jclass c, jlong ctx, jintArray inputTypes, jintArray groups, jintArray aggKinds, jobjectArray aggCols,
                              jintArray filterArgs, jlong expectedGroups, jobjectArray derived, jlongArray rowFilter) {
    gsql_agg_spec s;
    fill_agg_spec(env, &s, inputTypes, groups, aggKinds, aggCols, filterArgs, expectedGroups);
    s.n_derived = derived ? (*env)->GetArrayLength(env, derived) : 0;
    if (s.n_derived > GSQL_MAX_DERIVED) s.n_derived = GSQL_MAX_DERIVED;
    for (int i = 0; i < s.n_derived; i++) {
        int32_t d[4] = {0, 0, 0, 0}, nd;
        jintArray one = (jintArray)(*env)->GetObjectArrayElement(env, derived, i);
        fill_ints(env, one, d, &nd, 4);
        (*env)->DeleteLocalRef(env, one);
        s.derived[i].kind = d[0];
        s.derived[i].a = d[1];
        s.derived[i].b = d[2];
        s.derived[i].c = d[3];
    }
    if (rowFilter) {
        jlong f[3];
        (*env)->GetLongArrayRegion(env, rowFilter, 0, 3, f);
        s.row_filter_col = (int32_t)f[0];
        s.row_filter_op = (int32_t)f[1];
        s.row_filter_value = f[2];
    }
    return agg_create(env, ctx, &s);
}

NATIVE(void, aggConsume)(JNIEnv *env, jclass c, jlong ah, jlong sh) {
    jhandle *h = (jhandle *)(intptr_t)ah;
    int st = gsql_agg_consume((gsql_agg *)h->h, as_batch((staging *)(intptr_t)sh, 0));
    if (st != GSQL_OK) throw_status(env, h->ctx, st);
}

NATIVE(jlong, aggFinish)(JNIEnv *env, jclass c, jlong ah) {
    jhandle *h = (jhandle *)(intptr_t)ah;
    int64_t groups = 0;
    int st = gsql_agg_finish((gsql_agg *)h->h, &groups);
    if (st != GSQL_OK) throw_status(env, h->ctx, st);
    return (jlong)groups;
}

NATIVE(jint, aggNext)(JNIEnv *env, jclass c, jlong ah, jlong oh, jint maxRows) {
    jhandle *h = (jhandle *)(intptr_t)ah;
    staging *o = (staging *)(intptr_t)oh;
    int64_t rows = 0;
    if (staging_reserve(o, maxRows)) { throw_status(env, NULL, GSQL_E_OOM); return -1; }
    int st = gsql_agg_next((gsql_agg *)h->h, as_batch(o, 1), maxRows, &rows);
    if (st != GSQL_OK) { throw_status(env, h->ctx, st); return -1; }
    staging_filled(o, rows);
    return (jint)rows;
}

NATIVE(void, aggDestroy)(JNIEnv *env, jclass c, jlong ah) {
    jhandle *h = (jhandle *)(intptr_t)ah;
    if (!h) return;
    gsql_agg_destroy((gsql_agg *)h->h);
    free(h);
}

/* ---- grouping sets: HashAgg over Expand (gsql_gsagg_*) ------------------------------------------------------ */
/* projSrc / projCol / projValue: one array per projection, one entry per Expand output column (gsql_expand_item). */
NATIVE(jlong, gsAggCreate)(JNIEnv *env, jclass c, jlong ctx, jintArray inputTypes, jintArray outputTypes, jobjectArray projSrc,
                           jobjectArray projCol, jobjectArray projValue, jintArray groups, jintArray aggKinds, jobjectArray aggCols,
                           jintArray filterArgs, jlong expectedGroups) {
    gsql_agg_spec s;
    fill_agg_spec(env, &s, outputTypes, groups, aggKinds, aggCols, filterArgs, expectedGroups);
    gsql_expand_spec *ep = (gsql_expand_spec *)calloc(1, sizeof(gsql_expand_spec)); /* 8 KB: off the JNI thread's stack */
    if (!ep) { throw_status(env, NULL, GSQL_E_OOM); return 0; }
    fill_ints(env, inputTypes, ep->input_types, &ep->n_input_cols, GSQL_MAX_COLS);
    ep->n_output_cols = s.n_input_cols;
    ep->nsets = projSrc ? (*env)->GetArrayLength(env, projSrc) : 0;
    for (int p = 0; p < ep->nsets && p < GSQL_MAX_SETS; p++) {
        int32_t src[GSQL_MAX_COLS], col[GSQL_MAX_COLS], ns = 0, nc = 0;
        jintArray a = (jintArray)(*env)->GetObjectArrayElement(env, projSrc, p);
        jintArray b = (jintArray)(*env)->GetObjectArrayElement(env, projCol, p);
        jlongArray v = (jlongArray)(*env)->GetObjectArrayElement(env, projValue, p);
        fill_ints(env, a, src, &ns, GSQL_MAX_COLS);
        fill_ints(env, b, col, &nc, GSQL_MAX_COLS);
        jlong vals[GSQL_MAX_COLS];
        jsize nv = v ? (*env)->GetArrayLength(env, v) : 0;
        if (nv > GSQL_MAX_COLS) nv = GSQL_MAX_COLS;
        if (nv) (*env)->GetLongArrayRegion(env, v, 0, nv, vals);
        for (int k = 0; k < ns; k++) {
            ep->proj[p][k].src = src[k];
            ep->proj[p][k].col = k < nc ? col[k] : -1;
            ep->proj[p][k].value = k < nv ? vals[k] : 0;
        }
        (*env)->DeleteLocalRef(env, a);
        (*env)->DeleteLocalRef(env, b);
        if (v) (*env)->DeleteLocalRef(env, v);
    }
    gsql_gsagg *g = NULL;
    int st = gsql_gsagg_create((gsql_ctx *)(intptr_t)ctx, ep, &s, &g);
    free(ep);
    if (st != GSQL_OK) { throw_status(env, (gsql_ctx *)(intptr_t)ctx, st); return 0; }
    jhandle *h = (jhandle *)calloc(1, sizeof(jhandle));
    h->ctx = (gsql_ctx *)(intptr_t)ctx;
    h->h = g;
    return (jlong)(intptr_t)h;
}

NATIVE(void, gsAggConsume)(JNIEnv *env, jclass c, jlong ah, jlong sh) {
    jhandle *h = (jhandle *)(intptr_t)ah;
    int st = gsql_gsagg_consume((gsql_gsagg *)h->h, as_batch((staging *)(intptr_t)sh, 0));
    if (st != GSQL_OK) throw_status(env, h->ctx, st);
}

NATIVE(jlong, gsAggFinish)(JNIEnv *env, jclass c, jlong ah) {
    jhandle *h = (jhandle *)(intptr_t)ah;
    int64_t groups = 0;
    int st = gsql_gsagg_finish((gsql_gsagg *)h->h, &groups);
    if (st != GSQL_OK) throw_status(env, h->ctx, st);
    return (jlong)groups;
}

NATIVE(jint, gsAggNext)(JNIEnv *env, jclass c, jlong ah, jlong oh, jint maxRows) {
    jhandle *h = (jhandle *)(intptr_t)ah;
    staging *o = (staging *)(intptr_t)oh;
    int64_t rows = 0;
    if (staging_reserve(o, maxRows)) { throw_status(env, NULL, GSQL_E_OOM); return -1; }
    int st = gsql_gsagg_next((gsql_gsagg *)h->h, as_batch(o, 1), maxRows, &rows);
    if (st != GSQL_OK) { throw_status(env, h->ctx, st); return -1; }
    staging_filled(o, rows);
    return (jint)rows;
}

NATIVE(void, gsAggDestroy)(JNIEnv *env, jclass c, jlong ah) {
    jhandle *h = (jhandle *)(intptr_t)ah;
    if (!h) return;
    gsql_gsagg_destroy((gsql_gsagg *)h->h);
    free(h);
}

/* ---- sorted aggregation (gsql_sortagg_*) -------------------------------------------------------------------- */
NATIVE(jlong, sortAggCreate)(JNIEnv *env, jclass c, jlong ctx, jintArray inputTypes, jintArray groups, jintArray aggKinds,
                             jobjectArray aggCols, jintArray filterArgs) {
    gsql_agg_spec s;
    fill_agg_spec(env, &s, inputTypes, groups, aggKinds, aggCols, filterArgs, 0);
    gsql_sortagg *a = NULL;
    int st = gsql_sortagg_create((gsql_ctx *)(intptr_t)ctx, &s, &a);
    if (st != GSQL_OK) { throw_status(env, (gsql_ctx *)(intptr_t)ctx, st); return 0; }
    jhandle *h = (jhandle *)calloc(1, sizeof(jhandle));
    h->ctx = (gsql_ctx *)(intptr_t)ctx;
    h->h = a;
    return (jlong)(intptr_t)h;
}

/* returns the groups ready to be returned */
NATIVE(jlong, sortAggConsume)(JNIEnv *env, jclass c, jlong ah, jlong sh) {
    jhandle *h = (jhandle *)(intptr_t)ah;
    int64_t ready = 0;
    int st = gsql_sortagg_consume((gsql_sortagg *)h->h, as_batch((staging *)(intptr_t)sh, 0), &ready);
    if (st != GSQL_OK) { throw_status(env, h->ctx, st); return -1; }
    return (jlong)ready;
}

NATIVE(jlong, sortAggFinish)(JNIEnv *env, jclass c, jlong ah) {
    jhandle *h = (jhandle *)(intptr_t)ah;
    int64_t ready = 0;
    int st = gsql_sortagg_finish((gsql_sortagg *)h->h, &ready);
    if (st != GSQL_OK) { throw_status(env, h->ctx, st); return -1; }
    return (jlong)ready;
}

NATIVE(jint, sortAggNext)(JNIEnv *env, jclass c, jlong ah, jlong oh, jint maxRows) {
    jhandle *h = (jhandle *)(intptr_t)ah;
    staging *o = (staging *)(intptr_t)oh;
    int64_t rows = 0;
    if (staging_reserve(o, maxRows)) { throw_status(env, NULL, GSQL_E_OOM); return -1; }
    int st = gsql_sortagg_next((gsql_sortagg *)h->h, as_batch(o, 1), maxRows, &rows);
    if (st != GSQL_OK) { throw_status(env, h->ctx, st); return -1; }
    staging_filled(o, rows);
    return (jint)rows;
}

NATIVE(void, sortAggDestroy)(JNIEnv *env, jclass c, jlong ah) {
    jhandle *h = (jhandle *)(intptr_t)ah;
    if (!h) return;
    gsql_sortagg_destroy((gsql_sortagg *)h->h);
    free(h);
}

/* ---- sort-merge join (gsql_smj_*) ----------------------------------------------------------------------------- */
NATIVE(jlong, smjCreate)(JNIEnv *env, jclass c, jlong ctx, jint joinType, jboolean maxOneRow, jintArray outerKeys, jintArray innerKeys,
                         jintArray keyTypes, jintArray keyDesc, jintArray outerTypes, jintArray innerTypes, jintArray antiOperands) {
    gsql_join_spec s;
    memset(&s, 0, sizeof(s));
    int32_t n, desc[GSQL_MAX_KEYS] = {0};
    /* one entry per key in every key array, at most GSQL_MAX_KEYS keys: anything else would be truncated or read short */
    const jsize nk = outerKeys ? (*env)->GetArrayLength(env, outerKeys) : 0;
    if (nk < 1 || nk > GSQL_MAX_KEYS || !innerKeys || !keyTypes || !keyDesc || (*env)->GetArrayLength(env, innerKeys) != nk ||
        (*env)->GetArrayLength(env, keyTypes) != nk || (*env)->GetArrayLength(env, keyDesc) != nk) {
        throw_status(env, NULL, GSQL_E_INVALID);
        return 0;
    }
    s.join_type = joinType;
    s.max_one_row = maxOneRow;
    fill_ints(env, outerKeys, s.outer_key, &s.nkeys, GSQL_MAX_KEYS);
    fill_ints(env, innerKeys, s.inner_key, &n, GSQL_MAX_KEYS);
    fill_ints(env, keyTypes, s.key_type, &n, GSQL_MAX_KEYS);
    fill_ints(env, keyDesc, desc, &n, GSQL_MAX_KEYS);
    fill_ints(env, outerTypes, s.outer_types, &s.n_outer_cols, GSQL_MAX_COLS);
    fill_ints(env, innerTypes, s.inner_types, &s.n_inner_cols, GSQL_MAX_COLS);
    fill_ints(env, antiOperands, s.anti_operands, &s.n_anti_operands, GSQL_MAX_KEYS);
    gsql_smj *j = NULL;
    int st = gsql_smj_create((gsql_ctx *)(intptr_t)ctx, &s, desc, &j);
    if (st != GSQL_OK) { throw_status(env, (gsql_ctx *)(intptr_t)ctx, st); return 0; }
    jhandle *h = (jhandle *)calloc(1, sizeof(jhandle));
    h->ctx = (gsql_ctx *)(intptr_t)ctx;
    h->h = j;
    return (jlong)(intptr_t)h;
}

NATIVE(void, smjInnerConsume)(JNIEnv *env, jclass c, jlong jh, jlong sh) {
    jhandle *h = (jhandle *)(intptr_t)jh;
    int st = gsql_smj_inner_consume((gsql_smj *)h->h, as_batch((staging *)(intptr_t)sh, 0));
    if (st != GSQL_OK) throw_status(env, h->ctx, st);
}

NATIVE(void, smjInnerFinish)(JNIEnv *env, jclass c, jlong jh) {
    jhandle *h = (jhandle *)(intptr_t)jh;
    int st = gsql_smj_inner_finish((gsql_smj *)h->h);
    if (st != GSQL_OK) throw_status(env, h->ctx, st);
}

/* a host batch is uploaded by the library, so the staging may be reset as soon as this returns */
NATIVE(jlong, smjProbe)(JNIEnv *env, jclass c, jlong jh, jlong sh) {
    jhandle *h = (jhandle *)(intptr_t)jh;
    int64_t rows = 0;
    int st = gsql_smj_probe((gsql_smj *)h->h, as_batch((staging *)(intptr_t)sh, 0), &rows);
    if (st != GSQL_OK) { throw_status(env, h->ctx, st); return -1; }
    return (jlong)rows;
}

NATIVE(jint, smjNext)(JNIEnv *env, jclass c, jlong jh, jlong oh, jint maxRows) {
    jhandle *h = (jhandle *)(intptr_t)jh;
    staging *o = (staging *)(intptr_t)oh;
    int64_t rows = 0;
    if (staging_reserve(o, maxRows)) { throw_status(env, NULL, GSQL_E_OOM); return -1; }
    int st = gsql_smj_next((gsql_smj *)h->h, as_batch(o, 1), maxRows, &rows);
    if (st != GSQL_OK) { throw_status(env, h->ctx, st); return -1; }
    staging_filled(o, rows);
    return (jint)rows;
}

NATIVE(void, smjDestroy)(JNIEnv *env, jclass c, jlong jh) {
    jhandle *h = (jhandle *)(intptr_t)jh;
    if (!h) return;
    gsql_smj_destroy((gsql_smj *)h->h);
    free(h);
}

/* ---- window (gsql_window_*): NonFrameOverWindowExec -------------------------------------------------------- */
NATIVE(jlong, windowCreate)(JNIEnv *env, jclass c, jlong ctx, jintArray inputTypes, jintArray partition, jintArray callKinds,
                            jobjectArray callCols, jintArray filterArgs, jboolean resetEachRow) {
    gsql_window_spec s;
    memset(&s, 0, sizeof(s));
    int32_t kinds[GSQL_MAX_AGGS], fargs[GSQL_MAX_AGGS], n;
    fill_ints(env, inputTypes, s.input_types, &s.n_input_cols, GSQL_MAX_COLS);
    fill_ints(env, partition, s.part_cols, &s.npart, GSQL_MAX_KEYS);
    fill_ints(env, callKinds, kinds, &s.ncalls, GSQL_MAX_AGGS);
    fill_ints(env, filterArgs, fargs, &n, GSQL_MAX_AGGS);
    for (int i = 0; i < s.ncalls; i++) {
        jintArray cols = callCols ? (jintArray)(*env)->GetObjectArrayElement(env, callCols, i) : NULL;
        s.calls[i].kind = kinds[i];
        s.calls[i].filter_arg = i < n ? fargs[i] : -1;
        fill_ints(env, cols, s.calls[i].cols, &s.calls[i].ncols, 4);
        if (cols && (*env)->GetArrayLength(env, cols) > 4) s.calls[i].ncols = 5; /* refused by the library: more than 4 columns */
        if (cols) (*env)->DeleteLocalRef(env, cols);
    }
    s.reset_each_row = resetEachRow ? 1 : 0;
    gsql_window *w = NULL;
    int st = gsql_window_create((gsql_ctx *)(intptr_t)ctx, &s, &w);
    if (st != GSQL_OK) { throw_status(env, (gsql_ctx *)(intptr_t)ctx, st); return 0; }
    jhandle *h = (jhandle *)calloc(1, sizeof(jhandle));
    h->ctx = (gsql_ctx *)(intptr_t)ctx;
    h->h = w;
    return (jlong)(intptr_t)h;
}

/* the staged input rows -> one row per input row in outStaging's call columns; returns the row count */
NATIVE(jint, windowApply)(JNIEnv *env, jclass c, jlong wh, jlong sh, jlong oh) {
    jhandle *h = (jhandle *)(intptr_t)wh;
    staging *in = (staging *)(intptr_t)sh;
    staging *o = (staging *)(intptr_t)oh;
    if (staging_reserve(o, in->rows)) { throw_status(env, NULL, GSQL_E_OOM); return -1; }
    int st = gsql_window_apply((gsql_window *)h->h, as_batch(in, 0), as_batch(o, 1));
    if (st != GSQL_OK) { throw_status(env, h->ctx, st); return -1; }
    staging_filled(o, in->rows);
    return (jint)in->rows;
}

NATIVE(void, windowDestroy)(JNIEnv *env, jclass c, jlong wh) {
    jhandle *h = (jhandle *)(intptr_t)wh;
    if (!h) return;
    gsql_window_destroy((gsql_window *)h->h);
    free(h);
}

/* ---- vectorised filter / project ---------------------------------------------------------------------------- */
static int fill_expr(JNIEnv *env, gsql_expr *e, jintArray ops, jintArray args, jlongArray consts) {
    int32_t o[GSQL_MAX_EXPR_INS], a[GSQL_MAX_EXPR_INS], n, m;
    jlong k[GSQL_MAX_EXPR_INS];
    memset(e, 0, sizeof(*e));
    fill_ints(env, ops, o, &n, GSQL_MAX_EXPR_INS);
    fill_ints(env, args, a, &m, GSQL_MAX_EXPR_INS);
    if (m != n || !consts || (*env)->GetArrayLength(env, consts) < n) return -1;
    (*env)->GetLongArrayRegion(env, consts, 0, n, k);
    e->n = n;
    for (int i = 0; i < n; i++) {
        e->ins[i].op = o[i];
        e->ins[i].arg = a[i];
        e->ins[i].k.i = k[i]; /* doubles travel as Double.doubleToRawLongBits */
    }
    return 0;
}

NATIVE(jlong, scanCreate)(JNIEnv *env, jclass c, jlong ctx, jintArray inputTypes, jintArray filterOps, jintArray filterArgs, jlongArray filterConsts,
                          jobjectArray outOps, jobjectArray outArgs, jobjectArray outConsts) {
    gsql_scan_spec *s = (gsql_scan_spec *)calloc(1, sizeof(gsql_scan_spec));
    int bad = 0;
    fill_ints(env, inputTypes, s->input_types, &s->n_input_cols, GSQL_MAX_COLS);
    s->has_filter = filterOps != NULL;
    if (s->has_filter) bad |= fill_expr(env, &s->filter, filterOps, filterArgs, filterConsts);
    s->n_out = outOps ? (*env)->GetArrayLength(env, outOps) : 0;
    if (s->n_out > GSQL_MAX_SCAN_OUT) bad = 1;
    for (int i = 0; i < s->n_out && !bad; i++) {
        jintArray o = (jintArray)(*env)->GetObjectArrayElement(env, outOps, i);
        jintArray a = (jintArray)(*env)->GetObjectArrayElement(env, outArgs, i);
        jlongArray k = (jlongArray)(*env)->GetObjectArrayElement(env, outConsts, i);
        bad |= fill_expr(env, &s->out[i], o, a, k);
        (*env)->DeleteLocalRef(env, o);
        (*env)->DeleteLocalRef(env, a);
        (*env)->DeleteLocalRef(env, k);
    }
    gsql_scan *sc = NULL;
    int st = bad ? GSQL_E_INVALID : gsql_scan_create((gsql_ctx *)(intptr_t)ctx, s, &sc);
    free(s);
    if (st != GSQL_OK) { throw_status(env, bad ? NULL : (gsql_ctx *)(intptr_t)ctx, st); return 0; }
    jhandle *h = (jhandle *)calloc(1, sizeof(jhandle));
    h->ctx = (gsql_ctx *)(intptr_t)ctx;
    h->h = sc;
    return (jlong)(intptr_t)h;
}

NATIVE(jint, scanApply)(JNIEnv *env, jclass c, jlong sh, jlong ih, jlong oh) {
    jhandle *h = (jhandle *)(intptr_t)sh;
    staging *in = (staging *)(intptr_t)ih, *o = (staging *)(intptr_t)oh;
    int64_t rows = 0;
    if (staging_reserve(o, in->rows)) { throw_status(env, NULL, GSQL_E_OOM); return -1; }
    int st = gsql_scan_apply((gsql_scan *)h->h, as_batch(in, 0), as_batch(o, 1), o->cap, &rows);
    if (st != GSQL_OK) { throw_status(env, h->ctx, st); return -1; }
    staging_filled(o, rows);
    return (jint)rows;
}

NATIVE(void, scanDestroy)(JNIEnv *env, jclass c, jlong sh) {
    jhandle *h = (jhandle *)(intptr_t)sh;
    if (!h) return;
    gsql_scan_destroy((gsql_scan *)h->h);
    free(h);
}

/* ---- local hash-partition exchange -------------------------------------------------------------------------- */
/* ---- PagesSerde wire format (gsql_serde_*): a staging batch <-> the framed page stream of PagesSerdeUtil.writeSerializedChunk */
NATIVE(jbyteArray, serdeSerialize)(JNIEnv *env, jclass c, jlong ctx, jlong sh, jint pageRows) {
    staging *in = (staging *)(intptr_t)sh;
    gsql_ctx *cx = (gsql_ctx *)(intptr_t)ctx;
    int64_t need = 0, got = 0;
    int st = gsql_serde_size(cx, as_batch(in, 0), pageRows, &need);
    if (st != GSQL_OK) { throw_status(env, cx, st); return NULL; }
    if (need > 0x7fffffff) { throw_status(env, NULL, GSQL_E_CAPACITY); return NULL; } /* a Java byte[] holds 2^31 - 1 bytes */
    void *buf = NULL;
    if (gsql_host_alloc((size_t)(need ? need : 1), &buf) != GSQL_OK) { throw_status(env, NULL, GSQL_E_OOM); return NULL; }
    st = gsql_serde_serialize(cx, as_batch(in, 0), pageRows, buf, need, &got);
    jbyteArray out = NULL;
    if (st != GSQL_OK) {
        throw_status(env, cx, st);
    } else {
        out = (*env)->NewByteArray(env, (jsize)got);
        if (out) (*env)->SetByteArrayRegion(env, out, 0, (jsize)got, (const jbyte *)buf);
    }
    gsql_host_free(buf);
    return out;
}

NATIVE(jint, serdeDeserialize)(JNIEnv *env, jclass c, jlong ctx, jbyteArray pages, jint offset, jint length, jlong oh) {
    staging *o = (staging *)(intptr_t)oh;
    gsql_ctx *cx = (gsql_ctx *)(intptr_t)ctx;
    if (!pages || offset < 0 || length < 0 || offset + (int64_t)length > (*env)->GetArrayLength(env, pages)) { throw_status(env, NULL, GSQL_E_INVALID); return -1; }
    void *buf = NULL;
    if (gsql_host_alloc((size_t)(length ? length : 1), &buf) != GSQL_OK) { throw_status(env, NULL, GSQL_E_OOM); return -1; }
    (*env)->GetByteArrayRegion(env, pages, offset, length, (jbyte *)buf);
    int64_t rows = 0;
    /* first call learns the row count when the staging batch is too small (GSQL_E_CAPACITY reports the need) */
    int st = gsql_serde_deserialize(cx, buf, length, GSQL_MEM_HOST, as_batch(o, 1), o->cap, &rows);
    if (st == GSQL_E_CAPACITY && rows > o->cap) {
        if (staging_reserve(o, rows)) { gsql_host_free(buf); throw_status(env, NULL, GSQL_E_OOM); return -1; }
        st = gsql_serde_deserialize(cx, buf, length, GSQL_MEM_HOST, as_batch(o, 1), o->cap, &rows);
    }
    gsql_host_free(buf);
    if (st != GSQL_OK) { throw_status(env, cx, st); return -1; }
    staging_filled(o, rows);
    return (jint)rows;
}

NATIVE(jlong, xchgCreate)(JNIEnv *env, jclass c, jlong ctx, jintArray types, jintArray channels, jintArray keyTypes, jint nparts, jint mode) {
    gsql_xchg_spec s;
    int32_t n;
    memset(&s, 0, sizeof(s));
    fill_ints(env, types, s.types, &s.n_cols, GSQL_MAX_COLS);
    fill_ints(env, channels, s.channels, &s.n_channels, GSQL_MAX_KEYS);
    fill_ints(env, keyTypes, s.key_types, &n, GSQL_MAX_KEYS);
    s.nparts = nparts;
    s.mode = mode;
    gsql_xchg *x = NULL;
    int st = gsql_xchg_create((gsql_ctx *)(intptr_t)ctx, &s, &x);
    if (st != GSQL_OK) { throw_status(env, (gsql_ctx *)(intptr_t)ctx, st); return 0; }
    jhandle *h = (jhandle *)calloc(1, sizeof(jhandle));
    h->ctx = (gsql_ctx *)(intptr_t)ctx;
    h->h = x;
    return (jlong)(intptr_t)h;
}

NATIVE(void, xchgPartition)(JNIEnv *env, jclass c, jlong xh, jlong ih, jlong oh, jlongArray partCounts) {
    jhandle *h = (jhandle *)(intptr_t)xh;
    staging *in = (staging *)(intptr_t)ih, *o = (staging *)(intptr_t)oh;
    int64_t counts[GSQL_MAX_PARTS];
    if (staging_reserve(o, in->rows)) { throw_status(env, NULL, GSQL_E_OOM); return; }
    gsql_batch *ib = as_batch(in, 0), *ob = as_batch(o, 1);
    for (int i = 0; i < in->ncols; i++) /* the partitioned copy carries a mask exactly where the input does */
        if (!ib->cols[i].nulls) ob->cols[i].nulls = NULL;
    int st = gsql_xchg_partition((gsql_xchg *)h->h, ib, ob, counts);
    if (st != GSQL_OK) { throw_status(env, h->ctx, st); return; }
    o->rows = in->rows;
    for (int i = 0; i < in->ncols; i++) o->any_null[i] = in->any_null[i];
    jsize n = (*env)->GetArrayLength(env, partCounts);
    (*env)->SetLongArrayRegion(env, partCounts, 0, n, (const jlong *)counts);
}

NATIVE(void, xchgDestroy)(JNIEnv *env, jclass c, jlong xh) {
    jhandle *h = (jhandle *)(intptr_t)xh;
    if (!h) return;
    gsql_xchg_destroy((gsql_xchg *)h->h);
    free(h);
}

/* ---- runtime bloom filter (gsql_bloom_*): RuntimeFilterBuilderExec / FilterExec BLOOMFILTER(key) ----------------- */
/* the handle remembers the bitmap's size: a Java long[] that does not hold exactly that many words is rejected here,
 * before any byte is copied (the library trusts its callers' buffer sizes) */
typedef struct jbloom {
    gsql_ctx *ctx;
    gsql_bloom *b;
    int64_t nwords; /* num_bits / 64 */
} jbloom;

static void throw_invalid(JNIEnv *env, const char *msg) {
    if ((*env)->ExceptionCheck(env)) return;
    (*env)->ThrowNew(env, (*env)->FindClass(env, "com/alibaba/polardbx/executor/operator/gpu/GpuExecutorException"), msg);
}

NATIVE(jlong, bloomCreate)(JNIEnv *env, jclass c, jlong ctx, jlong numBits, jint numHashFunctions) {
    gsql_bloom *b = NULL;
    int st = gsql_bloom_create((gsql_ctx *)(intptr_t)ctx, numBits, numHashFunctions, &b);
    if (st != GSQL_OK) { throw_status(env, (gsql_ctx *)(intptr_t)ctx, st); return 0; }
    jbloom *h = (jbloom *)calloc(1, sizeof(jbloom));
    h->ctx = (gsql_ctx *)(intptr_t)ctx;
    h->b = b;
    h->nwords = numBits / 64;
    return (jlong)(intptr_t)h;
}

NATIVE(void, bloomPut)(JNIEnv *env, jclass c, jlong bh, jlong sh, jint keyCol) {
    jbloom *h = (jbloom *)(intptr_t)bh;
    int st = gsql_bloom_put(h->b, as_batch((staging *)(intptr_t)sh, 0), keyCol);
    if (st != GSQL_OK) throw_status(env, h->ctx, st);
}

/* words: nfilters bitmaps back to back (BloomFilter.getBitmap() of each, e.g. BloomFilterConsume's), ORed into the filter;
 * words.length must be nfilters * num_bits / 64 */
NATIVE(void, bloomMerge)(JNIEnv *env, jclass c, jlong bh, jlongArray words, jint nfilters) {
    jbloom *h = (jbloom *)(intptr_t)bh;
    if (!words || nfilters < 1 || (int64_t)(*env)->GetArrayLength(env, words) != (int64_t)nfilters * h->nwords) {
        throw_invalid(env, "bloomMerge: words must hold nfilters bitmaps of exactly num_bits / 64 longs each");
        return;
    }
    const jsize n = (*env)->GetArrayLength(env, words);
    void *buf = NULL;
    if (gsql_host_alloc((size_t)n * 8, &buf) != GSQL_OK) { throw_status(env, NULL, GSQL_E_OOM); return; }
    (*env)->GetLongArrayRegion(env, words, 0, n, (jlong *)buf);
    int st = gsql_bloom_merge(h->b, (const uint64_t *)buf, nfilters, GSQL_MEM_HOST);
    gsql_host_free(buf);
    if (st != GSQL_OK) throw_status(env, h->ctx, st);
}

/* words |= the GPU bitmap: the caller holds the shared BloomFilter's lock and passes its getBitmap() array, which must
 * hold exactly num_bits / 64 longs */
NATIVE(void, bloomBitmapOr)(JNIEnv *env, jclass c, jlong bh, jlongArray words) {
    jbloom *h = (jbloom *)(intptr_t)bh;
    if (!words || (int64_t)(*env)->GetArrayLength(env, words) != h->nwords) {
        throw_invalid(env, "bloomBitmapOr: words must hold exactly num_bits / 64 longs");
        return;
    }
    const jsize n = (jsize)h->nwords;
    void *buf = NULL;
    if (gsql_host_alloc((size_t)n * 8, &buf) != GSQL_OK) { throw_status(env, NULL, GSQL_E_OOM); return; }
    int st = gsql_bloom_bitmap(h->b, (uint64_t *)buf, GSQL_MEM_HOST);
    if (st == GSQL_OK) {
        jlong *w = (jlong *)(*env)->GetPrimitiveArrayCritical(env, words, NULL);
        if (w) {
            for (jsize i = 0; i < n; i++) w[i] |= ((const jlong *)buf)[i];
            (*env)->ReleasePrimitiveArrayCritical(env, words, w, 0);
        } else {
            st = GSQL_E_OOM;
        }
    }
    gsql_host_free(buf);
    if (st != GSQL_OK) throw_status(env, h->ctx, st);
}

NATIVE(jint, bloomFilter)(JNIEnv *env, jclass c, jlong bh, jlong ih, jint keyCol, jlong oh) {
    jbloom *h = (jbloom *)(intptr_t)bh;
    staging *in = (staging *)(intptr_t)ih, *o = (staging *)(intptr_t)oh;
    int64_t rows = 0;
    if (staging_reserve(o, in->rows)) { throw_status(env, NULL, GSQL_E_OOM); return -1; }
    int st = gsql_bloom_filter(h->b, as_batch(in, 0), keyCol, as_batch(o, 1), o->cap, &rows);
    if (st != GSQL_OK) { throw_status(env, h->ctx, st); return -1; }
    staging_filled(o, rows);
    return (jint)rows;
}

NATIVE(void, bloomDestroy)(JNIEnv *env, jclass c, jlong bh) {
    jbloom *h = (jbloom *)(intptr_t)bh;
    if (!h) return;
    gsql_bloom_destroy(h->b);
    free(h);
}

/* ---- ORDER BY / TOP-N ------------------------------------------------------------------------------------------ */
/* gsql_sort_spec from the Java arrays; 0, or -1 with GSQL_E_INVALID thrown */
static int sort_spec(JNIEnv *env, jintArray types, jintArray keyCols, jintArray keyDesc, jlong limit, gsql_sort_spec *s) {
    int32_t nd = 0;
    memset(s, 0, sizeof(*s));
    /* longer arrays than the spec holds are refused, not truncated: a dropped sort key would change the order */
    if ((types && (*env)->GetArrayLength(env, types) > GSQL_MAX_COLS) || (keyCols && (*env)->GetArrayLength(env, keyCols) > GSQL_MAX_KEYS) ||
        (keyDesc && (*env)->GetArrayLength(env, keyDesc) > GSQL_MAX_KEYS)) {
        throw_status(env, NULL, GSQL_E_INVALID);
        return -1;
    }
    fill_ints(env, types, s->types, &s->n_cols, GSQL_MAX_COLS);
    fill_ints(env, keyCols, s->key_col, &s->nkeys, GSQL_MAX_KEYS);
    fill_ints(env, keyDesc, s->key_desc, &nd, GSQL_MAX_KEYS);
    if (nd != s->nkeys) {
        throw_status(env, NULL, GSQL_E_INVALID);
        return -1;
    }
    s->limit = limit;
    return 0;
}

NATIVE(jlong, sortCreate)(JNIEnv *env, jclass c, jlong ctx, jintArray types, jintArray keyCols, jintArray keyDesc, jlong limit) {
    gsql_sort_spec s;
    if (sort_spec(env, types, keyCols, keyDesc, limit, &s)) return 0;
    gsql_sort *so = NULL;
    int st = gsql_sort_create((gsql_ctx *)(intptr_t)ctx, &s, &so);
    if (st != GSQL_OK) { throw_status(env, (gsql_ctx *)(intptr_t)ctx, st); return 0; }
    jhandle *h = (jhandle *)calloc(1, sizeof(jhandle));
    h->ctx = (gsql_ctx *)(intptr_t)ctx;
    h->h = so;
    return (jlong)(intptr_t)h;
}

NATIVE(void, sortConsume)(JNIEnv *env, jclass c, jlong sh, jlong stg) {
    jhandle *h = (jhandle *)(intptr_t)sh;
    int st = gsql_sort_consume((gsql_sort *)h->h, as_batch((staging *)(intptr_t)stg, 0));
    if (st != GSQL_OK) throw_status(env, h->ctx, st);
}

NATIVE(jlong, sortFinish)(JNIEnv *env, jclass c, jlong sh) {
    jhandle *h = (jhandle *)(intptr_t)sh;
    int64_t rows = 0;
    int st = gsql_sort_finish((gsql_sort *)h->h, &rows);
    if (st != GSQL_OK) throw_status(env, h->ctx, st);
    return (jlong)rows;
}

NATIVE(jint, sortNext)(JNIEnv *env, jclass c, jlong sh, jlong oh, jint maxRows) {
    jhandle *h = (jhandle *)(intptr_t)sh;
    staging *o = (staging *)(intptr_t)oh;
    int64_t rows = 0;
    if (staging_reserve(o, maxRows)) { throw_status(env, NULL, GSQL_E_OOM); return -1; }
    int st = gsql_sort_next((gsql_sort *)h->h, as_batch(o, 1), maxRows, &rows);
    if (st != GSQL_OK) { throw_status(env, h->ctx, st); return -1; }
    staging_filled(o, rows);
    return (jint)rows;
}

NATIVE(void, sortDestroy)(JNIEnv *env, jclass c, jlong sh) {
    jhandle *h = (jhandle *)(intptr_t)sh;
    if (!h) return;
    gsql_sort_destroy((gsql_sort *)h->h);
    free(h);
}

/* ---- merge of sorted runs (MergeSortExec) ----------------------------------------------------------------------- */
NATIVE(jlong, mergeCreate)(JNIEnv *env, jclass c, jlong ctx, jintArray types, jintArray keyCols, jintArray keyDesc, jint nInputs,
                           jlong limit) {
    gsql_sort_spec s;
    if (sort_spec(env, types, keyCols, keyDesc, limit, &s)) return 0;
    gsql_merge *m = NULL;
    int st = gsql_merge_create((gsql_ctx *)(intptr_t)ctx, &s, nInputs, &m);
    if (st != GSQL_OK) { throw_status(env, (gsql_ctx *)(intptr_t)ctx, st); return 0; }
    jhandle *h = (jhandle *)calloc(1, sizeof(jhandle));
    h->ctx = (gsql_ctx *)(intptr_t)ctx;
    h->h = m;
    return (jlong)(intptr_t)h;
}

NATIVE(void, mergeConsume)(JNIEnv *env, jclass c, jlong mh, jint input, jlong stg) {
    jhandle *h = (jhandle *)(intptr_t)mh;
    int st = gsql_merge_consume((gsql_merge *)h->h, input, as_batch((staging *)(intptr_t)stg, 0));
    if (st != GSQL_OK) throw_status(env, h->ctx, st);
}

NATIVE(jlong, mergeFinish)(JNIEnv *env, jclass c, jlong mh) {
    jhandle *h = (jhandle *)(intptr_t)mh;
    int64_t rows = 0;
    int st = gsql_merge_finish((gsql_merge *)h->h, &rows);
    if (st != GSQL_OK) throw_status(env, h->ctx, st);
    return (jlong)rows;
}

NATIVE(jint, mergeNext)(JNIEnv *env, jclass c, jlong mh, jlong oh, jint maxRows) {
    jhandle *h = (jhandle *)(intptr_t)mh;
    staging *o = (staging *)(intptr_t)oh;
    int64_t rows = 0;
    if (staging_reserve(o, maxRows)) { throw_status(env, NULL, GSQL_E_OOM); return -1; }
    int st = gsql_merge_next((gsql_merge *)h->h, as_batch(o, 1), maxRows, &rows);
    if (st != GSQL_OK) { throw_status(env, h->ctx, st); return -1; }
    staging_filled(o, rows);
    return (jint)rows;
}

NATIVE(void, mergeDestroy)(JNIEnv *env, jclass c, jlong mh) {
    jhandle *h = (jhandle *)(intptr_t)mh;
    if (!h) return;
    gsql_merge_destroy((gsql_merge *)h->h);
    free(h);
}
