// smj.cuh — SortMergeJoinExec behind gsql_smj_* (included from sort.cu for MAX_ROW_IDS and is_null).
//
// Reference path replaced: EX/operator/SortMergeJoinExec.java (the two-pointer walk, :186-278; JoinResultsIterator,
// :375-455; the NOT IN check on the first inner row, :559-567) and AbstractJoinExec.java:79-134 (output schema, anti
// operands).  The walk's output for key-ordered inputs is restated per outer row, which is what makes it parallel:
//   * keys are converted to their unified type (gsql_load_key) and compared key by key by NumberType.compare, negated
//     under DESC: two NULLs are equal and NULL is the smallest value; doubles by Double.compareTo (-0.0 < +0.0, every NaN
//     equal, above +Inf);
//   * an outer row whose keys hold no NULL is matched by the run of inner rows with equal keys, if there is one;
//   * rows come out in outer order; a matched row is followed by its run in inner order (INNER / LEFT / RIGHT), once
//     (SEMI), or not at all (ANTI); an unmatched row gives one NULL-padded row (LEFT / RIGHT) or itself (ANTI, when its
//     anti operands are all non-NULL or the inner side is empty);
//   * single join: one row per matched outer row; a run of two or more rows is GSQL_E_MORE_THAN_ONE_ROW.
// Each key becomes an order image: the unified value's u64 image (the sort's value_image mapping), complemented under DESC,
// below a rank bit that puts NULL first under ASC and last under DESC (rank[r] bit k).  Images are not range-compressed:
// outer batches arrive after the inner side is fixed, so one encoding must cover values not yet seen.
//   finish:  k_smj_image + k_smj_order (inner order check, run heads) -> cub inclusive scan (run ids) -> k_smj_run_end;
//   probe:   k_smj_image + k_smj_order (outer order check, also against the previous batch's last row, k_smj_keep_last)
//            -> k_smj_match (each CTA bounds the inner window of its 1024 outer rows with two full lower-bound searches,
//            then every row searches inside the window: ordered outer rows read the inner images about once) -> cub
//            exclusive scan of the per-row output counts (64-bit offsets, the exact total);
//   next:    k_smj_expand (a CTA bounds the outer rows of its 1024 output rows the same way over the offsets; each thread
//            gathers one output row, stores are coalesced per column).
#include <cub/device/device_scan.cuh>

namespace {

constexpr int SJ_THREADS = 256;
constexpr int SJ_RPT = 4;
constexpr int SJ_TILE = SJ_THREADS * SJ_RPT;
constexpr int64_t SJ_MAX_OUTER_BATCH = INT32_MAX - 1;  // the scan covers n + 1 counts, and cub's item count is an int

struct SmjKeys {  // the key columns of one side, their unified types and directions
    int32_t nk;
    uint32_t asc_mask;  // bit k: key k is ascending
    DCol c[GSQL_MAX_KEYS];
    int32_t utype[GSQL_MAX_KEYS];
};

struct SmjImages {  // img[k * n + r]: the order image of key k at row r; rank[r] bit k: key k's NULL rank bit
    const uint64_t *img;
    const uint8_t *rank;
    int64_t n;
};

// Order image of a non-NULL unified value: value_image's mapping applied after gsql_load_key's conversion.
__device__ __forceinline__ uint64_t smj_value_image(const KeyVal &k, int utype) {
    if (utype == GSQL_T_INT32) return (uint64_t)(int64_t)(int32_t)k.i ^ (1ULL << 63);
    if (utype == GSQL_T_INT64) return (uint64_t)k.i ^ (1ULL << 63);
    const uint64_t b = (uint64_t)k.i;
    const uint64_t canon = ((b & 0x7fffffffffffffffULL) > 0x7ff0000000000000ULL) ? 0x7ff8000000000000ULL : b;
    return (canon >> 63) ? ~canon : (canon | (1ULL << 63));
}

// (rank bit, image) per key, compared lexicographically, is the comparator: a NULL has image 0 and rank 0 under ASC
// (below every value, whose rank is 1) and rank 1 under DESC (above every value, whose rank is 0 and image complemented).
__global__ void __launch_bounds__(SJ_THREADS) k_smj_image(const __grid_constant__ SmjKeys K, int64_t n, uint64_t *__restrict__ img,
                                                          uint8_t *__restrict__ rank) {
    for (int64_t r = blockIdx.x * (int64_t)blockDim.x + threadIdx.x; r < n; r += (int64_t)gridDim.x * blockDim.x) {
        uint32_t rk = 0;
#pragma unroll 1
        for (int k = 0; k < K.nk; k++) {
            const KeyVal v = gsql_load_key(K.c[k], r, K.utype[k]);
            const bool asc = (K.asc_mask >> k) & 1u;
            uint64_t x = 0;
            if (!v.is_null) x = asc ? smj_value_image(v, K.utype[k]) : ~smj_value_image(v, K.utype[k]);
            if (asc != v.is_null) rk |= 1u << k;
            img[(int64_t)k * n + r] = x;
        }
        rank[r] = (uint8_t)rk;
    }
}

__device__ __forceinline__ int smj_cmp(const SmjImages &A, int64_t a, const SmjImages &B, int64_t b, int nk) {
    const uint32_t ra = A.rank[a], rb = B.rank[b];
#pragma unroll 1
    for (int k = 0; k < nk; k++) {
        const uint32_t x = (ra >> k) & 1u, y = (rb >> k) & 1u;
        if (x != y) return x < y ? -1 : 1;
        const uint64_t u = A.img[(int64_t)k * A.n + a], v = B.img[(int64_t)k * B.n + b];
        if (u != v) return u < v ? -1 : 1;
    }
    return 0;
}

// bad[0] = 1 when a row sorts before its predecessor (row 0's predecessor is prev's one row, when prev.n == 1).
// head (may be null): head[r] = 1 when row r starts a run of equal keys.
__global__ void __launch_bounds__(SJ_THREADS) k_smj_order(const SmjImages S, int nk, const SmjImages prev, uint32_t *__restrict__ head,
                                                          int32_t *__restrict__ bad) {
    bool unordered = false;
    for (int64_t r = blockIdx.x * (int64_t)blockDim.x + threadIdx.x; r < S.n; r += (int64_t)gridDim.x * blockDim.x) {
        const int c = r > 0 ? smj_cmp(S, r - 1, S, r, nk) : (prev.n ? smj_cmp(prev, 0, S, 0, nk) : -1);
        unordered |= c > 0;
        if (head) head[r] = (r == 0 || c != 0) ? 1u : 0u;
    }
    if (__syncthreads_or(unordered) && threadIdx.x == 0) bad[0] = 1;
}

// dst (one row, nk keys) = the last row of S.
__global__ void k_smj_keep_last(const SmjImages S, int nk, uint64_t *__restrict__ dst_img, uint8_t *__restrict__ dst_rank) {
    for (int k = 0; k < nk; k++) dst_img[k] = S.img[(int64_t)k * S.n + S.n - 1];
    dst_rank[0] = S.rank[S.n - 1];
}

// run_end[run_id[r] - 1] = r + 1 for the last row r of every run (run_id: inclusive scan of the head flags).
__global__ void __launch_bounds__(SJ_THREADS) k_smj_run_end(const uint32_t *__restrict__ run_id, int64_t n, uint32_t *__restrict__ run_end) {
    for (int64_t r = blockIdx.x * (int64_t)blockDim.x + threadIdx.x; r < n; r += (int64_t)gridDim.x * blockDim.x)
        if (r == n - 1 || run_id[r + 1] != run_id[r]) run_end[run_id[r] - 1] = (uint32_t)(r + 1);
}

struct SmjMatch {
    int32_t nk;
    int32_t join_type;
    int32_t single;
    int32_t inner_empty;
    uint32_t null_of_rank;  // rank ^ null_of_rank has bit k set where key k is NULL (the ascending keys' bits)
    int32_t n_anti;
    DCol anti[GSQL_MAX_KEYS];  // the outer batch's anti-operand columns
};

// First inner row in [lo, hi) that does not sort before outer row o (hi if there is none).
__device__ __forceinline__ int64_t smj_lower_bound(const SmjImages &I, const SmjImages &O, int64_t o, int nk, int64_t lo, int64_t hi) {
    while (lo < hi) {
        const int64_t mid = (lo + hi) >> 1;
        if (smj_cmp(I, mid, O, o, nk) < 0) lo = mid + 1;
        else hi = mid;
    }
    return lo;
}

// Per outer row: lbm[o] = first row of its matching inner run, -1 when unmatched; cnt[o] = its output rows.
// flags[1] = 1: a single join's outer row matches two or more inner rows.
__global__ void __launch_bounds__(SJ_THREADS) k_smj_match(const SmjImages I, const uint32_t *__restrict__ run_id,
                                                          const uint32_t *__restrict__ run_end, const SmjImages O,
                                                          const __grid_constant__ SmjMatch M, int32_t *__restrict__ lbm,
                                                          int64_t *__restrict__ cnt, int32_t *__restrict__ flags) {
    __shared__ int64_t win[2];
    const int64_t ntiles = (O.n + SJ_TILE - 1) / SJ_TILE;
    const uint32_t key_mask = (1u << M.nk) - 1u;
    for (int64_t tile = blockIdx.x; tile < ntiles; tile += gridDim.x) {
        const int64_t t0 = tile * SJ_TILE, t1 = t0 + SJ_TILE < O.n ? t0 + SJ_TILE : O.n;
        if (threadIdx.x == 0) win[0] = smj_lower_bound(I, O, t0, M.nk, 0, I.n);
        if (threadIdx.x == 32) win[1] = smj_lower_bound(I, O, t1 - 1, M.nk, 0, I.n);
        __syncthreads();
        // Ordered outer rows have their lower bounds inside [win0, win1]; unordered ones only get a result that the
        // order check throws away, and every search stays inside the inner rows.
        const int64_t lo = win[0], hi = win[1] > lo ? win[1] : lo;
        bool violation = false;
#pragma unroll 1
        for (int s = 0; s < SJ_RPT; s++) {
            const int64_t o = t0 + s * SJ_THREADS + threadIdx.x;
            if (o >= t1) break;
            const int64_t lb = smj_lower_bound(I, O, o, M.nk, lo, hi);
            const bool key_null = ((O.rank[o] ^ M.null_of_rank) & key_mask) != 0;
            int64_t run = 0;
            if (!key_null && lb < I.n && smj_cmp(I, lb, O, o, M.nk) == 0) run = (int64_t)run_end[run_id[lb] - 1] - lb;
            const bool matched = run > 0;
            int64_t c;
            if (M.join_type == GSQL_JOIN_SEMI) {
                c = matched ? 1 : 0;
            } else if (M.join_type == GSQL_JOIN_ANTI) {
                bool ok = !matched;
                if (ok && !M.inner_empty)
                    for (int a = 0; a < M.n_anti; a++) ok = ok && !is_null(M.anti[a], o);
                c = ok ? 1 : 0;
            } else {
                c = matched ? (M.single ? 1 : run) : (M.join_type == GSQL_JOIN_INNER ? 0 : 1);
            }
            violation |= M.single && run > 1;
            lbm[o] = matched ? (int32_t)lb : -1;
            cnt[o] = c;
        }
        if (violation) flags[1] = 1;
        __syncthreads();  // win is rewritten by the next tile
    }
}

struct SmjOut {
    int32_t n;
    int32_t pad;
    int8_t side[GSQL_MAX_COLS * 2];  // 0: outer column, 1: inner column
    int8_t col[GSQL_MAX_COLS * 2];
    void *data[GSQL_MAX_COLS * 2];
    uint8_t *nulls[GSQL_MAX_COLS * 2];
};

// Last outer row in [lo, hi) whose output offset is at most i (off[lo] <= i).
__device__ __forceinline__ int64_t smj_row_of(const int64_t *off, int64_t i, int64_t lo, int64_t hi) {
    while (lo < hi) {
        const int64_t mid = (lo + hi) >> 1;
        if (off[mid] <= i) lo = mid + 1;
        else hi = mid;
    }
    return lo - 1;
}

__device__ __forceinline__ void smj_put(const DCol &c, int64_t r, void *data, uint8_t *nulls, int64_t w, int32_t *flags) {
    const bool nl = r < 0 || is_null(c, r);
    if (c.type == GSQL_T_INT32) reinterpret_cast<int *>(data)[w] = nl ? 0 : reinterpret_cast<const int *>(c.data)[r];
    else reinterpret_cast<long long *>(data)[w] = nl ? 0 : reinterpret_cast<const long long *>(c.data)[r];
    if (nulls) nulls[w] = nl ? 1 : 0;
    else if (nl) flags[0] = 1;
}

// Output rows [base, base + m) of the current outer batch into row 0.. of W.  flags[0] = 1: a NULL met a column without a
// nulls buffer.
__global__ void __launch_bounds__(SJ_THREADS) k_smj_expand(const __grid_constant__ DColSet OC, const __grid_constant__ DColSet IC,
                                                           const int64_t *__restrict__ off, const int32_t *__restrict__ lbm, int64_t nb,
                                                           int64_t base, int64_t m, const __grid_constant__ SmjOut W,
                                                           int32_t *__restrict__ flags) {
    __shared__ int64_t win[2];
    const int64_t ntiles = (m + SJ_TILE - 1) / SJ_TILE;
    for (int64_t tile = blockIdx.x; tile < ntiles; tile += gridDim.x) {
        const int64_t i0 = base + tile * SJ_TILE, i1 = i0 + SJ_TILE < base + m ? i0 + SJ_TILE : base + m;
        if (threadIdx.x == 0) win[0] = smj_row_of(off, i0, 0, nb);
        if (threadIdx.x == 32) win[1] = smj_row_of(off, i1 - 1, 0, nb);
        __syncthreads();
        const int64_t lo = win[0], hi = win[1] + 1;
#pragma unroll 1
        for (int s = 0; s < SJ_RPT; s++) {
            const int64_t i = i0 + s * SJ_THREADS + threadIdx.x;
            if (i >= i1) break;
            const int64_t o = smj_row_of(off, i, lo, hi);
            const int32_t lb = lbm[o];
            const int64_t ir = lb < 0 ? -1 : lb + (i - off[o]);
            const int64_t w = i - base;
#pragma unroll 1
            for (int e = 0; e < W.n; e++) {
                if (W.side[e] == 0) smj_put(OC.c[W.col[e]], o, W.data[e], W.nulls[e], w, flags);
                else smj_put(IC.c[W.col[e]], ir, W.data[e], W.nulls[e], w, flags);
            }
        }
        __syncthreads();
    }
}

}  // namespace

struct gsql_smj {
    gsql_ctx *ctx;
    gsql_join_spec spec;
    RowStore inner;
    uint32_t asc_mask = 0;
    int32_t nout = 0;
    int8_t out_side[GSQL_MAX_COLS * 2], out_col[GSQL_MAX_COLS * 2];
    int32_t out_types[GSQL_MAX_COLS * 2];
    bool single = false, finished = false, pass_nothing = false;
    int64_t n_in = 0;
    DevBuf in_img, in_rank, run_id, run_end;
    // the outer batch being returned: referenced (device) or uploaded (host) until next() returns 0 rows
    StagedBatch *outer = nullptr;
    DevBuf o_img, o_rank, lbm, off, scan_tmp;
    int64_t nb = 0, total = 0, cursor = 0;
    DevBuf prev_img, prev_rank;  // the last row of the previous outer batch
    bool have_prev = false;
    DevBuf flags;  // [0] NULL into a column without nulls, [1] single-join violation, [2] unordered rows

    ~gsql_smj() { delete outer; }
    void drop_outer() {
        delete outer;
        outer = nullptr;
        nb = total = cursor = 0;
    }
    SmjKeys keys_of(const DCol *cols, const int32_t *key_col) const {
        SmjKeys K;
        memset(&K, 0, sizeof(K));
        K.nk = spec.nkeys;
        K.asc_mask = asc_mask;
        for (int k = 0; k < spec.nkeys; k++) {
            K.c[k] = cols[key_col[k]];
            K.utype[k] = spec.key_type[k];
        }
        return K;
    }
};

namespace {

// Images of `n` rows' keys into img / rank, and the order check of those rows (after prev's row when given).
gsql_status smj_images(gsql_smj *j, const SmjKeys &K, int64_t n, DevBuf *img, DevBuf *rank, const SmjImages &prev, uint32_t *head,
                       bool *unordered) {
    gsql_ctx *ctx = j->ctx;
    GSQL_TRY(img->alloc(ctx, (size_t)n * K.nk * 8));
    GSQL_TRY(rank->alloc(ctx, (size_t)n));
    if (n == 0) {
        *unordered = false;
        return GSQL_OK;
    }
    {
        KernelScope ks(ctx, "k_smj_image");
        k_smj_image<<<grid_for(ctx, n, SJ_THREADS, 8), SJ_THREADS, 0, ctx->stream>>>(K, n, img->as<uint64_t>(), rank->as<uint8_t>());
    }
    GSQL_CUDA(ctx, cudaGetLastError());
    GSQL_CUDA(ctx, cudaMemsetAsync(j->flags.as<int32_t>() + 2, 0, 4, ctx->stream));
    {
        KernelScope ks(ctx, "k_smj_order");
        k_smj_order<<<grid_for(ctx, n, SJ_THREADS, 8), SJ_THREADS, 0, ctx->stream>>>(SmjImages{img->as<uint64_t>(), rank->as<uint8_t>(), n}, K.nk,
                                                                               prev, head, j->flags.as<int32_t>() + 2);
    }
    GSQL_CUDA(ctx, cudaGetLastError());
    int32_t bad = 0;
    GSQL_CUDA(ctx, cudaMemcpyAsync(&bad, j->flags.as<int32_t>() + 2, 4, cudaMemcpyDeviceToHost, ctx->stream));
    GSQL_CUDA(ctx, cudaStreamSynchronize(ctx->stream));
    *unordered = bad != 0;
    return GSQL_OK;
}

}  // namespace

extern "C" gsql_status gsql_smj_create(gsql_ctx *ctx, const gsql_join_spec *spec, const int32_t *key_desc, gsql_smj **out) {
    if (!ctx || !spec || !key_desc || !out) return GSQL_E_INVALID;
    *out = nullptr;
    if (ctx->sticky) return GSQL_E_CUDA;
    const gsql_join_spec &s = *spec;
    if (s.join_type < GSQL_JOIN_INNER || s.join_type > GSQL_JOIN_ANTI) return gsql_set_error(ctx, GSQL_E_INVALID, "join type %d", s.join_type);
    if (s.n_outer_cols < 1 || s.n_outer_cols > GSQL_MAX_COLS || s.n_inner_cols < 1 || s.n_inner_cols > GSQL_MAX_COLS)
        return gsql_set_error(ctx, GSQL_E_INVALID, "column counts %d / %d: must be in [1, %d]", s.n_outer_cols, s.n_inner_cols, GSQL_MAX_COLS);
    if (s.nkeys < 1 || s.nkeys > GSQL_MAX_KEYS) return gsql_set_error(ctx, GSQL_E_UNSUPPORTED, "nkeys %d: must be in [1, %d]", s.nkeys, GSQL_MAX_KEYS);
    if (s.n_cond != 0) return gsql_set_error(ctx, GSQL_E_UNSUPPORTED, "a join condition besides the keys (the stock operator keeps it)");
    if (s.build_outer) return gsql_set_error(ctx, GSQL_E_UNSUPPORTED, "build_outer: the merge join has no build side");
    if (s.max_one_row && s.join_type != GSQL_JOIN_INNER && s.join_type != GSQL_JOIN_LEFT)
        return gsql_set_error(ctx, GSQL_E_UNSUPPORTED, "single (max-one-row) join of type %d", s.join_type);
    for (int side = 0; side < 2; side++) {
        const int n = side ? s.n_inner_cols : s.n_outer_cols;
        const int32_t *t = side ? s.inner_types : s.outer_types;
        for (int i = 0; i < n; i++) {
            if (t[i] == GSQL_T_DEC128) return gsql_set_error(ctx, GSQL_E_UNSUPPORTED, "%s column %d: DEC128", side ? "inner" : "outer", i);
            if (t[i] < GSQL_T_INT32 || t[i] > GSQL_T_FP64) return gsql_set_error(ctx, GSQL_E_INVALID, "%s column %d: type %d", side ? "inner" : "outer", i, t[i]);
        }
    }
    for (int k = 0; k < s.nkeys; k++) {
        if (s.outer_key[k] < 0 || s.outer_key[k] >= s.n_outer_cols || s.inner_key[k] < 0 || s.inner_key[k] >= s.n_inner_cols)
            return gsql_set_error(ctx, GSQL_E_INVALID, "key %d out of range", k);
        if (s.key_type[k] == GSQL_T_DEC128) return gsql_set_error(ctx, GSQL_E_UNSUPPORTED, "key %d: DEC128", k);
        if (s.key_type[k] < GSQL_T_INT32 || s.key_type[k] > GSQL_T_FP64) return gsql_set_error(ctx, GSQL_E_INVALID, "key %d: type %d", k, s.key_type[k]);
        if (key_desc[k] != 0 && key_desc[k] != 1) return gsql_set_error(ctx, GSQL_E_INVALID, "key %d: key_desc %d is neither 0 nor 1", k, key_desc[k]);
    }
    if (s.n_anti_operands < 0 || s.n_anti_operands > GSQL_MAX_KEYS) return gsql_set_error(ctx, GSQL_E_INVALID, "n_anti_operands %d", s.n_anti_operands);
    for (int i = 0; i < s.n_anti_operands; i++)
        if (s.anti_operands[i] < 0 || s.anti_operands[i] >= s.n_outer_cols) return gsql_set_error(ctx, GSQL_E_INVALID, "anti operand %d out of range", i);
    GSQL_CUDA(ctx, cudaSetDevice(ctx->device));
    gsql_smj *j = new gsql_smj();
    j->ctx = ctx;
    gsql_ctx_retain(ctx);
    j->spec = s;
    j->inner.init(s.inner_types, s.n_inner_cols);
    j->single = s.max_one_row != 0;
    for (int k = 0; k < s.nkeys; k++)
        if (!key_desc[k]) j->asc_mask |= 1u << k;
    // output schema (AbstractJoinExec.java:102-118): semi / anti -> outer; single -> outer + inner[0]; RIGHT -> inner ||
    // outer; otherwise outer || inner
    auto push = [&](int side, int col) {
        j->out_side[j->nout] = (int8_t)side;
        j->out_col[j->nout] = (int8_t)col;
        j->out_types[j->nout] = side ? s.inner_types[col] : s.outer_types[col];
        j->nout++;
    };
    const bool semi = s.join_type == GSQL_JOIN_SEMI || s.join_type == GSQL_JOIN_ANTI;
    if (s.join_type == GSQL_JOIN_RIGHT)
        for (int i = 0; i < s.n_inner_cols; i++) push(1, i);
    for (int i = 0; i < s.n_outer_cols; i++) push(0, i);
    if (j->single) push(1, 0);
    else if (!semi && s.join_type != GSQL_JOIN_RIGHT)
        for (int i = 0; i < s.n_inner_cols; i++) push(1, i);
    gsql_status st = j->flags.alloc(ctx, 16);
    if (st == GSQL_OK) st = j->prev_img.alloc(ctx, GSQL_MAX_KEYS * 8);
    if (st == GSQL_OK) st = j->prev_rank.alloc(ctx, 16);
    if (st == GSQL_OK && cudaMemsetAsync(j->flags.p, 0, 16, ctx->stream) != cudaSuccess) st = GSQL_E_CUDA;
    if (st != GSQL_OK) {
        gsql_smj_destroy(j);
        return st;
    }
    *out = j;
    return GSQL_OK;
}

extern "C" void gsql_smj_destroy(gsql_smj *j) { destroy_handle(j); }

extern "C" gsql_status gsql_smj_inner_consume(gsql_smj *j, const gsql_batch *inner) {
    if (!j || !inner) return GSQL_E_INVALID;
    gsql_ctx *ctx = j->ctx;
    if (ctx->sticky) return GSQL_E_CUDA;
    if (j->finished) return gsql_set_error(ctx, GSQL_E_STATE, "inner_consume after inner_finish");
    GSQL_TRY(validate_batch(ctx, inner, j->spec.n_inner_cols, j->spec.inner_types));
    if (inner->rows == 0) return GSQL_OK;
    if (j->inner.rows + inner->rows > MAX_ROW_IDS)
        return gsql_set_error(ctx, GSQL_E_CAPACITY, "%lld inner rows exceed the 32-bit row ids (%lld)", (long long)(j->inner.rows + inner->rows),
                              (long long)MAX_ROW_IDS);
    GSQL_CUDA(ctx, cudaSetDevice(ctx->device));
    GSQL_TRY(j->inner.append(ctx, inner, inner->rows));
    if (inner->mem == GSQL_MEM_HOST) GSQL_CUDA(ctx, cudaStreamSynchronize(ctx->stream));  // the caller may reuse its buffers
    return GSQL_OK;
}

extern "C" gsql_status gsql_smj_inner_finish(gsql_smj *j) {
    if (!j) return GSQL_E_INVALID;
    gsql_ctx *ctx = j->ctx;
    if (ctx->sticky) return GSQL_E_CUDA;
    if (j->finished) return gsql_set_error(ctx, GSQL_E_STATE, "inner_finish called twice");
    GSQL_CUDA(ctx, cudaSetDevice(ctx->device));
    const int64_t n = j->inner.rows;
    const DColSet v = j->inner.view();
    bool unordered = false;
    DevBuf head;
    GSQL_TRY(head.alloc(ctx, (size_t)n * 4));
    GSQL_TRY(smj_images(j, j->keys_of(v.c, j->spec.inner_key), n, &j->in_img, &j->in_rank, SmjImages{nullptr, nullptr, 0}, head.as<uint32_t>(),
                        &unordered));
    if (unordered) return gsql_set_error(ctx, GSQL_E_INVALID, "inner rows are not ordered on the join keys");
    GSQL_TRY(j->run_id.alloc(ctx, (size_t)n * 4));
    GSQL_TRY(j->run_end.alloc(ctx, (size_t)n * 4));
    if (n > 0) {
        size_t need = 0;
        GSQL_CUDA(ctx, cub::DeviceScan::InclusiveSum(nullptr, need, head.as<uint32_t>(), j->run_id.as<uint32_t>(), (int)n, ctx->stream));
        GSQL_TRY(j->scan_tmp.alloc(ctx, need));
        {
            KernelScope ks(ctx, "k_smj_runs");
            GSQL_CUDA(ctx, cub::DeviceScan::InclusiveSum(j->scan_tmp.p, need, head.as<uint32_t>(), j->run_id.as<uint32_t>(), (int)n, ctx->stream));
        }
        {
            KernelScope ks(ctx, "k_smj_run_end");
            k_smj_run_end<<<grid_for(ctx, n, SJ_THREADS, 8), SJ_THREADS, 0, ctx->stream>>>(j->run_id.as<uint32_t>(), n, j->run_end.as<uint32_t>());
        }
        GSQL_CUDA(ctx, cudaGetLastError());
        // NOT IN whose first inner row holds a NULL key produces nothing (doSpecialCheckForAntiJoin)
        if (j->spec.join_type == GSQL_JOIN_ANTI && j->spec.n_anti_operands > 0) {
            uint8_t r0 = 0;
            GSQL_CUDA(ctx, cudaMemcpyAsync(&r0, j->in_rank.p, 1, cudaMemcpyDeviceToHost, ctx->stream));
            GSQL_CUDA(ctx, cudaStreamSynchronize(ctx->stream));
            j->pass_nothing = ((r0 ^ j->asc_mask) & ((1u << j->spec.nkeys) - 1u)) != 0;
        }
    }
    GSQL_CUDA(ctx, cudaStreamSynchronize(ctx->stream));
    j->scan_tmp.release();
    j->n_in = n;
    j->finished = true;
    return GSQL_OK;
}

extern "C" gsql_status gsql_smj_output_schema(gsql_smj *j, int32_t *ncols, int32_t *types) {
    if (!j || !ncols) return GSQL_E_INVALID;
    return output_schema(j->nout, j->out_types, ncols, types);
}

extern "C" gsql_status gsql_smj_probe(gsql_smj *j, const gsql_batch *outer, int64_t *out_rows) {
    if (!j || !outer || !out_rows) return GSQL_E_INVALID;
    gsql_ctx *ctx = j->ctx;
    if (ctx->sticky) return GSQL_E_CUDA;
    *out_rows = 0;
    if (!j->finished) return gsql_set_error(ctx, GSQL_E_STATE, "probe before inner_finish");
    if (j->outer && j->cursor < j->total)
        return gsql_set_error(ctx, GSQL_E_STATE, "probe while %lld rows of the previous outer batch are still to be returned",
                              (long long)(j->total - j->cursor));
    GSQL_TRY(validate_batch(ctx, outer, j->spec.n_outer_cols, j->spec.outer_types));
    if (outer->rows > SJ_MAX_OUTER_BATCH)
        return gsql_set_error(ctx, GSQL_E_CAPACITY, "outer batch of %lld rows: at most %lld per probe", (long long)outer->rows,
                              (long long)SJ_MAX_OUTER_BATCH);
    GSQL_CUDA(ctx, cudaSetDevice(ctx->device));
    j->drop_outer();
    const int64_t n = outer->rows;
    if (n == 0 || j->pass_nothing) return GSQL_OK;
    StagedBatch *sb = new StagedBatch();
    const gsql_status st0 = stage_batch(ctx, outer, sb);
    if (st0 != GSQL_OK) {
        delete sb;
        return st0;
    }
    j->outer = sb;
    auto fail = [&](gsql_status st) {
        j->drop_outer();
        return st;
    };
    bool unordered = false;
    const SmjImages prev{j->prev_img.as<uint64_t>(), j->prev_rank.as<uint8_t>(), j->have_prev ? 1 : 0};
    gsql_status st = smj_images(j, j->keys_of(sb->cols, j->spec.outer_key), n, &j->o_img, &j->o_rank, prev, nullptr, &unordered);
    if (st != GSQL_OK) return fail(st);
    if (unordered)
        return fail(gsql_set_error(ctx, GSQL_E_INVALID, "outer rows are not ordered on the join keys (within the batch or after the previous batch)"));
    SmjMatch M;
    memset(&M, 0, sizeof(M));
    M.nk = j->spec.nkeys;
    M.join_type = j->spec.join_type;
    M.single = j->single;
    M.inner_empty = j->n_in == 0;
    M.null_of_rank = j->asc_mask;
    M.n_anti = j->spec.n_anti_operands;
    for (int a = 0; a < M.n_anti; a++) M.anti[a] = sb->cols[j->spec.anti_operands[a]];
    if ((st = j->lbm.alloc(ctx, (size_t)n * 4)) != GSQL_OK) return fail(st);
    if ((st = j->off.alloc(ctx, (size_t)(n + 1) * 8)) != GSQL_OK) return fail(st);
    DevBuf cnt;
    if ((st = cnt.alloc(ctx, (size_t)(n + 1) * 8)) != GSQL_OK) return fail(st);
    GSQL_CUDA(ctx, cudaMemsetAsync(cnt.as<int64_t>() + n, 0, 8, ctx->stream));
    GSQL_CUDA(ctx, cudaMemsetAsync(j->flags.p, 0, 16, ctx->stream));
    {
        KernelScope ks(ctx, "k_smj_match");
        k_smj_match<<<grid_for(ctx, n, SJ_TILE, 8), SJ_THREADS, 0, ctx->stream>>>(
            SmjImages{j->in_img.as<uint64_t>(), j->in_rank.as<uint8_t>(), j->n_in}, j->run_id.as<uint32_t>(), j->run_end.as<uint32_t>(),
            SmjImages{j->o_img.as<uint64_t>(), j->o_rank.as<uint8_t>(), n}, M, j->lbm.as<int32_t>(), cnt.as<int64_t>(), j->flags.as<int32_t>());
    }
    GSQL_CUDA(ctx, cudaGetLastError());
    size_t need = 0;
    GSQL_CUDA(ctx, cub::DeviceScan::ExclusiveSum(nullptr, need, cnt.as<int64_t>(), j->off.as<int64_t>(), (int)(n + 1), ctx->stream));
    if (!j->scan_tmp.p || need > j->scan_tmp.bytes)
        if ((st = j->scan_tmp.alloc(ctx, need)) != GSQL_OK) return fail(st);
    need = j->scan_tmp.bytes;
    {
        KernelScope ks(ctx, "k_smj_scan");
        GSQL_CUDA(ctx, cub::DeviceScan::ExclusiveSum(j->scan_tmp.p, need, cnt.as<int64_t>(), j->off.as<int64_t>(), (int)(n + 1), ctx->stream));
    }
    int32_t hf[4];
    int64_t total = 0;
    GSQL_CUDA(ctx, cudaMemcpyAsync(hf, j->flags.p, 16, cudaMemcpyDeviceToHost, ctx->stream));
    GSQL_CUDA(ctx, cudaMemcpyAsync(&total, j->off.as<int64_t>() + n, 8, cudaMemcpyDeviceToHost, ctx->stream));
    GSQL_CUDA(ctx, cudaStreamSynchronize(ctx->stream));
    if (hf[1]) {
        GSQL_CUDA(ctx, cudaMemsetAsync(j->flags.p, 0, 16, ctx->stream));
        return fail(gsql_set_error(ctx, GSQL_E_MORE_THAN_ONE_ROW, "single join: an outer row matches more than one inner row"));
    }
    {
        KernelScope ks(ctx, "k_smj_keep_last");
        k_smj_keep_last<<<1, 1, 0, ctx->stream>>>(SmjImages{j->o_img.as<uint64_t>(), j->o_rank.as<uint8_t>(), n}, j->spec.nkeys,
                                                  j->prev_img.as<uint64_t>(), j->prev_rank.as<uint8_t>());
    }
    GSQL_CUDA(ctx, cudaGetLastError());
    j->have_prev = true;
    j->nb = n;
    j->total = total;
    j->cursor = 0;
    *out_rows = total;
    return GSQL_OK;
}

extern "C" gsql_status gsql_smj_next(gsql_smj *j, gsql_batch *out, int64_t max_rows, int64_t *out_rows) {
    if (!j || !out || !out_rows) return GSQL_E_INVALID;
    gsql_ctx *ctx = j->ctx;
    if (ctx->sticky) return GSQL_E_CUDA;
    *out_rows = 0;
    if (!j->finished) return gsql_set_error(ctx, GSQL_E_STATE, "next before inner_finish");
    if (max_rows < 0) return gsql_set_error(ctx, GSQL_E_INVALID, "max_rows %lld < 0", (long long)max_rows);
    GSQL_TRY(validate_batch(ctx, out, j->nout, j->out_types));
    out->rows = 0;
    GSQL_CUDA(ctx, cudaSetDevice(ctx->device));
    const int64_t left = j->total - j->cursor;
    if (left == 0) {  // the batch is exhausted: a referenced device batch is no longer read
        j->drop_outer();
        return GSQL_OK;
    }
    const int64_t n = left < max_rows ? left : max_rows;
    if (n == 0) return GSQL_OK;
    OutBinding ob;
    GSQL_TRY(out_bind(ctx, out, n, &ob));
    SmjOut W;
    memset(&W, 0, sizeof(W));
    W.n = j->nout;
    for (int e = 0; e < j->nout; e++) {
        W.side[e] = j->out_side[e];
        W.col[e] = j->out_col[e];
        W.data[e] = ob.data[e];
        W.nulls[e] = ob.nulls[e];
    }
    const DColSet oc = j->outer->set(), ic = j->inner.view();
    {
        KernelScope ks(ctx, "k_smj_expand");
        k_smj_expand<<<grid_for(ctx, n, SJ_TILE, 8), SJ_THREADS, 0, ctx->stream>>>(oc, ic, j->off.as<int64_t>(), j->lbm.as<int32_t>(), j->nb,
                                                                              j->cursor, n, W, j->flags.as<int32_t>());
    }
    GSQL_CUDA(ctx, cudaGetLastError());
    int32_t hf[4];
    GSQL_CUDA(ctx, cudaMemcpyAsync(hf, j->flags.p, 16, cudaMemcpyDeviceToHost, ctx->stream));
    GSQL_CUDA(ctx, cudaStreamSynchronize(ctx->stream));
    if (hf[0]) {
        GSQL_CUDA(ctx, cudaMemsetAsync(j->flags.p, 0, 16, ctx->stream));
        return gsql_set_error(ctx, GSQL_E_INVALID, "a NULL had to be written into an output column without a nulls buffer");
    }
    GSQL_TRY(out_download(ctx, out, n, ob));
    j->cursor += n;
    *out_rows = out->rows = n;
    return GSQL_OK;
}
