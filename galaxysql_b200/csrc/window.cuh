// window.cuh — GPU NonFrameOverWindowExec behind gsql_window_* (included at the end of agg.cu, after agg_sorted.cuh; reuses
// its SState, sa_zero and sa_combine, and agg.cu's init_value, dbl_sortable / dbl_unsortable and agg_out_type).
//
// Reference path replaced (EX/ = polardbx-executor/src/main/java/com/alibaba/polardbx/executor/):
//   EX/operator/NonFrameOverWindowExec.java:79-146 (processFirstLine, doNextChunk, isDifferentPartition)
//   EX/calc/aggfunctions/RowNumber.java, Rank.java (sameRank: Objects.equals), DenseRank.java
//   EX/mpp/operator/factory/OverWindowFramesExecFactory.java:127-164 (which calls reach the operator, the reset frame)
//
// Every call's value at a row is an inclusive segmented scan over the rows: a segment starts at each partition head (every
// row with reset_each_row), and the scan element is the call's state over a run of rows, SState:
//   ROW_NUMBER  l = rows                           DENSE_RANK  l = peer heads
//   RANK        l = rows, x = rows up to and including the last peer head, has = the run holds a peer head
//   aggregates  sa_add's state of the rows (one row: sa_zero folded with the row's value)
// combined as (f1, a) + (f2, b) = (f1 | f2, f2 ? b : a o b).  Peer heads are the partition heads plus the rows whose RANK
// columns differ from the previous row's; comparing with the previous row rather than with the run's first row (as Rank
// does) is the same thing, Objects.equals being an equivalence.
//
// One kernel per batch, k_win_tile: one CTA per tile of WT_TILE rows, WT_IPT consecutive rows per thread.  Each column a
// step needs is staged into shared memory with coalesced cp.async copies (thread j copies rows j, j + WT_THREADS, ...;
// byte copies when a base is not aligned to its element), with the row before the tile in slot 0 (the carried row for tile
// 0).  Per call: a block scan of the threads' partials, chained across tiles by a decoupled look-back (one ScanTileState per
// call), seeded at tile 0 with the state carried from the previous batch.  The finished values go through shared memory
// and are stored with coalesced stores.  k_win_carry then keeps the batch's last row's keys and states for the next batch.

namespace {

constexpr int WT_THREADS = 256, WT_IPT = 4, WT_TILE = WT_THREADS * WT_IPT;
constexpr int WT_CARRY_KEYS = GSQL_MAX_KEYS + 4 * GSQL_MAX_AGGS;  // partition columns, then 4 RANK columns per call

struct WinCall {
    int32_t kind, in_type, out_type, ncols;
    int32_t cols[4];
};

struct WinOut {
    void *data;
    uint8_t *nulls;
};

struct WinParams {
    DColSet in;
    int64_t rows;
    int32_t ntiles, ncalls, npart, reset, has_carry, pad;
    int32_t part_col[GSQL_MAX_KEYS];
    WinCall call[GSQL_MAX_AGGS];
    WinOut out[GSQL_MAX_AGGS];
    const int64_t *ckey;   // [WT_CARRY_KEYS] the previous batch's last row: INT32 widened, DOUBLE as raw bits
    const uint8_t *cnull;  // [WT_CARRY_KEYS]
    const SState *cstate;  // [ncalls] the previous batch's last row's states
    SState *last;          // [ncalls] this batch's last row's states
    cub::ScanTileState<SState> tiles[GSQL_MAX_AGGS];
};

__device__ __forceinline__ bool win_rank_kind(int k) { return k == GSQL_AGG_RANK || k == GSQL_AGG_DENSE_RANK; }

// a then b, b holding no segment head
__device__ __forceinline__ SState win_combine(int kind, int in_type, const SState &a, const SState &b) {
    SState s = a;
    switch (kind) {
    case GSQL_AGG_ROW_NUMBER: case GSQL_AGG_DENSE_RANK: s.l = a.l + b.l; return s;
    case GSQL_AGG_RANK:
        s.l = a.l + b.l;
        s.x = b.has ? a.l + b.x : a.x;
        s.has = a.has | b.has;
        return s;
    default: return sa_combine<false>(kind, in_type, a, b);
    }
}

struct WinSegOp {
    int kind, in_type;
    __device__ __forceinline__ SState operator()(const SState &a, const SState &b) const {
        SState o = b.f ? b : win_combine(kind, in_type, a, b);
        o.f = a.f | b.f;
        return o;
    }
};

struct WinStage {  // one staged column: slot 0 = the row before the tile, slot 1 + j = row t0 + j
    alignas(16) unsigned char v[(WT_TILE + 1) * 8];
    uint8_t n[WT_TILE + 1];
};

// Stages column c's rows [t0, t0 + nlive) (values only when `values`) and the row before them.  Begins with a barrier (the
// previous readers of the stage are done) and ends with one (the stage is complete).
__device__ __forceinline__ void win_stage(WinStage &st, const DCol &c, int64_t t0, int nlive, bool values, bool carried,
                                          int64_t ckey, uint8_t cnull) {
    const int w = c.type == GSQL_T_INT32 ? 4 : 8;
    __syncthreads();
    if (values) {
        const unsigned char *src = reinterpret_cast<const unsigned char *>(c.data) + t0 * w;
        if ((reinterpret_cast<uintptr_t>(c.data) & (uintptr_t)(w - 1)) == 0) {
            for (int j = threadIdx.x; j < nlive; j += WT_THREADS) {
                if (w == 8) cp_async_8(st.v + (j + 1) * w, src + (int64_t)j * w);
                else cp_async_4(st.v + (j + 1) * w, src + (int64_t)j * w);
            }
            cp_async_commit();
        } else {
            for (int j = threadIdx.x; j < nlive; j += WT_THREADS)
                for (int b = 0; b < w; b++) st.v[(j + 1) * w + b] = src[(int64_t)j * w + b];
        }
    }
    for (int j = threadIdx.x; j < nlive; j += WT_THREADS) st.n[j + 1] = c.nulls ? __ldcs(c.nulls + t0 + j) : 0;
    if (threadIdx.x == 0) {
        if (t0 > 0) {
            st.n[0] = c.nulls ? c.nulls[t0 - 1] : 0;
            if (values) {
                const unsigned char *p = reinterpret_cast<const unsigned char *>(c.data) + (t0 - 1) * w;
                for (int b = 0; b < w; b++) st.v[b] = p[b];
            }
        } else if (carried) {
            st.n[0] = cnull;
            if (w == 4) reinterpret_cast<int *>(st.v)[0] = (int)ckey;
            else reinterpret_cast<long long *>(st.v)[0] = ckey;
        }
    }
    if (values) cp_async_wait<0>();
    __syncthreads();
}

__device__ __forceinline__ long long win_val(const WinStage &st, int type, int i) {
    return type == GSQL_T_INT32 ? (long long)reinterpret_cast<const int *>(st.v)[i] : reinterpret_cast<const long long *>(st.v)[i];
}

// Object.equals of slots i and j of a staged column (sa_key_eq's rule)
__device__ __forceinline__ bool win_eq(const WinStage &st, int type, int i, int j) {
    const bool ni = st.n[i] != 0, nj = st.n[j] != 0;
    if (ni || nj) return ni == nj;
    const long long a = win_val(st, type, i), b = win_val(st, type, j);
    if (type == GSQL_T_FP64) return gsql_double_bits(__longlong_as_double(a)) == gsql_double_bits(__longlong_as_double(b));
    return a == b;
}

// One row's state: sa_zero(kind) folded with the row (sa_add's rules); `v` is the value (raw bits for DOUBLE).
__device__ __forceinline__ SState win_row(const WinCall &cl, bool is_null, long long v) {
    SState s = sa_zero(cl.kind);
    switch (cl.kind) {
    case GSQL_AGG_COUNT_STAR: s.l = 1; return s;
    case GSQL_AGG_COUNT: s.l = is_null ? 0 : 1; return s;
    default: break;
    }
    if (is_null) return s;
    switch (cl.kind) {
    case GSQL_AGG_SUM:
        if (cl.in_type == GSQL_T_FP64) sa_set_d(s, __longlong_as_double(v) + 0.0);  // from +0.0: an all -0.0 sum is +0.0
        else {
            s.l = v;
            s.x = v < 0 ? -1 : 0;
        }
        s.has = 1;
        return s;
    case GSQL_AGG_AVG:
        sa_set_d(s, __longlong_as_double(v) + 0.0);
        s.l = 1;
        s.has = 1;
        return s;
    case GSQL_AGG_SUM0: s.l = v; return s;
    default: {  // MIN / MAX
        const bool mx = cl.kind == GSQL_AGG_MAX;
        s.l = cl.in_type == GSQL_T_FP64 ? dbl_sortable(__longlong_as_double(v), mx) : v;
        s.has = 1;
        return s;
    }
    }
}

// writeResultTo of a state: the value's words (lo, hi: DEC128 only) and the NULL flag (k_agg_finalize's rules)
__device__ __forceinline__ bool win_result(const WinCall &cl, const SState &s, long long &lo, long long &hi) {
    hi = 0;
    switch (cl.kind) {
    case GSQL_AGG_RANK: lo = s.x; return false;
    case GSQL_AGG_ROW_NUMBER: case GSQL_AGG_DENSE_RANK: case GSQL_AGG_COUNT_STAR: case GSQL_AGG_COUNT: case GSQL_AGG_SUM0:
        lo = s.l;
        return false;
    case GSQL_AGG_SUM:
        if (!s.has) { lo = 0; return true; }
        lo = cl.in_type == GSQL_T_FP64 ? s.x : s.l;
        hi = cl.in_type == GSQL_T_FP64 ? 0 : s.x;
        return false;
    case GSQL_AGG_AVG: {
        const bool ok = s.has && s.l != 0;
        lo = ok ? __double_as_longlong(sa_d(s) / (double)s.l) : 0;
        return !ok;
    }
    default:  // MIN / MAX
        if (!s.has) { lo = 0; return true; }
        lo = cl.in_type == GSQL_T_FP64 ? __double_as_longlong(dbl_unsortable(s.l, cl.kind == GSQL_AGG_MAX)) : s.l;
        return false;
    }
}

__global__ void k_win_init(const __grid_constant__ WinParams P) {
    for (int c = 0; c < P.ncalls; c++) {
        cub::ScanTileState<SState> ts = P.tiles[c];
        ts.InitializeStatus(P.ntiles);
    }
}

__global__ void __launch_bounds__(WT_THREADS) k_win_tile(const __grid_constant__ WinParams P) {
    typedef cub::BlockScan<SState, WT_THREADS> SegScan;
    typedef cub::TilePrefixCallbackOp<SState, WinSegOp, cub::ScanTileState<SState>> LookBack;
    __shared__ WinStage st;
    __shared__ struct {
        typename SegScan::TempStorage scan;
        typename LookBack::TempStorage lookback;
    } tmp;
    __shared__ alignas(16) long long ov[2 * WT_TILE];  // the call's values, row-major (two words a row for DEC128)
    __shared__ uint8_t on[WT_TILE];

    const int tile = blockIdx.x;
    const int64_t t0 = (int64_t)tile * WT_TILE;
    const int tile_rows = P.rows - t0 >= WT_TILE ? WT_TILE : (int)(P.rows - t0);
    const int r0 = threadIdx.x * WT_IPT;  // the thread's first row, tile-local
    const int nlive = tile_rows - r0 >= WT_IPT ? WT_IPT : (tile_rows > r0 ? tile_rows - r0 : 0);
    const unsigned live = (1u << nlive) - 1;
    const bool carried = P.has_carry != 0;

    // ---- partition heads: bit i = row r0 + i starts a partition
    unsigned head = 0;
    if (P.reset) {
        head = live;
    } else {
        if (tile == 0 && threadIdx.x == 0 && !carried) head |= 1u;
#pragma unroll 1
        for (int k = 0; k < P.npart; k++) {
            const DCol &c = P.in.c[P.part_col[k]];
            win_stage(st, c, t0, tile_rows, true, carried, carried ? P.ckey[k] : 0, carried ? P.cnull[k] : 0);
#pragma unroll
            for (int i = 0; i < WT_IPT; i++)
                if (i < nlive && !win_eq(st, c.type, r0 + i + 1, r0 + i)) head |= 1u << i;
        }
    }

    const int64_t last_row = P.rows - 1 - t0;  // tile-local index of the batch's last row (in this tile when < WT_TILE)
#pragma unroll 1
    for (int ci = 0; ci < P.ncalls; ci++) {
        const WinCall &cl = P.call[ci];
        SState e[WT_IPT];
        if (win_rank_kind(cl.kind)) {
            unsigned peer = head;
            if (!P.reset) {
#pragma unroll 1
                for (int q = 0; q < cl.ncols; q++) {
                    const DCol &c = P.in.c[cl.cols[q]];
                    const int slot = GSQL_MAX_KEYS + 4 * ci + q;
                    win_stage(st, c, t0, tile_rows, true, carried, carried ? P.ckey[slot] : 0, carried ? P.cnull[slot] : 0);
#pragma unroll
                    for (int i = 0; i < WT_IPT; i++)
                        if (i < nlive && !win_eq(st, c.type, r0 + i + 1, r0 + i)) peer |= 1u << i;
                }
            }
#pragma unroll
            for (int i = 0; i < WT_IPT; i++) {
                const bool p = (peer >> i) & 1u;
                e[i] = sa_zero(GSQL_AGG_COUNT_STAR);
                if (cl.kind == GSQL_AGG_DENSE_RANK) {
                    e[i].l = p ? 1 : 0;
                } else {
                    e[i].l = 1;
                    e[i].x = p ? 1 : 0;
                    e[i].has = p ? 1 : 0;
                }
            }
        } else if (cl.kind == GSQL_AGG_ROW_NUMBER || cl.kind == GSQL_AGG_COUNT_STAR) {
#pragma unroll
            for (int i = 0; i < WT_IPT; i++) {
                e[i] = sa_zero(GSQL_AGG_COUNT_STAR);
                e[i].l = 1;
            }
        } else if (cl.kind == GSQL_AGG_COUNT) {
            unsigned nul = 0;  // rows where a counted column is NULL
#pragma unroll 1
            for (int q = 0; q < cl.ncols; q++) {
                const DCol &c = P.in.c[cl.cols[q]];
                if (!c.nulls) continue;
                win_stage(st, c, t0, tile_rows, false, false, 0, 0);
#pragma unroll
                for (int i = 0; i < WT_IPT; i++)
                    if (st.n[r0 + i + 1]) nul |= 1u << i;
            }
#pragma unroll
            for (int i = 0; i < WT_IPT; i++) e[i] = win_row(cl, (nul >> i) & 1u, 0);
        } else {
            const DCol &c = P.in.c[cl.cols[0]];
            win_stage(st, c, t0, tile_rows, true, false, 0, 0);
#pragma unroll
            for (int i = 0; i < WT_IPT; i++) e[i] = win_row(cl, st.n[r0 + i + 1] != 0, win_val(st, c.type, r0 + i + 1));
        }
#pragma unroll
        for (int i = 0; i < WT_IPT; i++) e[i].f = (head >> i) & 1u;

        // the thread's partial, then the tile's scan chained to the earlier tiles'
        const WinSegOp op{cl.kind, cl.in_type};
        SState part = sa_zero(cl.kind);  // a right identity of op (f = 0, has = 0)
#pragma unroll
        for (int i = 0; i < WT_IPT; i++)
            if (i < nlive) part = op(part, e[i]);
        SState ex;
        __syncthreads();  // the previous call's scan storage and value stage are free again
        if (tile == 0) {
            SState seed = carried ? P.cstate[ci] : sa_zero(cl.kind), agg;
            seed.f = 0;
            SegScan(tmp.scan).ExclusiveScan(part, ex, seed, op, agg);
            if (threadIdx.x == 0) {
                cub::ScanTileState<SState> ts = P.tiles[ci];
                ts.SetInclusive(0, op(seed, agg));
            }
        } else {
            cub::ScanTileState<SState> ts = P.tiles[ci];
            LookBack prefix(ts, tmp.lookback, op, tile);
            SegScan(tmp.scan).ExclusiveScan(part, ex, op, prefix);
        }

        // per-row inclusive values into the stage
        const bool wide = cl.out_type == GSQL_T_DEC128;
        SState run = ex;
#pragma unroll
        for (int i = 0; i < WT_IPT; i++) {
            if (i < nlive) {
                run = op(run, e[i]);
                long long lo, hi;
                const bool n = win_result(cl, run, lo, hi);
                const int r = r0 + i;
                on[r] = n ? 1 : 0;
                if (wide) {
                    ov[2 * r] = lo;
                    ov[2 * r + 1] = hi;
                } else if (cl.out_type == GSQL_T_INT32) {
                    reinterpret_cast<int *>(ov)[r] = (int)lo;
                } else {
                    ov[r] = lo;
                }
                if (r == last_row) P.last[ci] = run;
            }
        }
        __syncthreads();

        // coalesced stores: thread j writes rows j, j + WT_THREADS, ...
        const WinOut &o = P.out[ci];
        for (int j = threadIdx.x; j < tile_rows; j += WT_THREADS) {
            __stcs(o.nulls + t0 + j, on[j]);
            if (wide) {
                long long *d = reinterpret_cast<long long *>(o.data) + 2 * (t0 + j);
                __stcs(d, ov[2 * j]);
                __stcs(d + 1, ov[2 * j + 1]);
            } else if (cl.out_type == GSQL_T_INT32) {
                __stcs(reinterpret_cast<int *>(o.data) + t0 + j, reinterpret_cast<const int *>(ov)[j]);
            } else {
                __stcs(reinterpret_cast<long long *>(o.data) + t0 + j, ov[j]);
            }
        }
    }
}

struct WinCarry {
    DColSet in;
    int64_t row;  // the batch's last row
    int32_t ncalls, nkeys;
    int32_t key_col[WT_CARRY_KEYS];  // -1: slot unused
    int64_t *ckey;
    uint8_t *cnull;
    SState *cstate;
    const SState *last;
};

// The last row's partition and RANK keys and every call's state, for the next batch's row 0.  The key is read byte by
// byte, as win_stage reads the row before a tile, so that a base not aligned to its element is read as well.
__global__ void k_win_carry(const __grid_constant__ WinCarry C) {
    for (int k = threadIdx.x; k < C.nkeys; k += blockDim.x) {
        if (C.key_col[k] < 0) continue;
        const DCol &c = C.in.c[C.key_col[k]];
        const int w = c.type == GSQL_T_INT32 ? 4 : 8;
        const unsigned char *p = reinterpret_cast<const unsigned char *>(c.data) + C.row * w;
        unsigned long long u = 0;
        for (int b = w - 1; b >= 0; b--) u = (u << 8) | p[b];
        const bool is_null = c.nulls != nullptr && c.nulls[C.row] != 0;
        C.ckey[k] = is_null ? 0 : (w == 4 ? (long long)(int)(unsigned)u : (long long)u);  // INT32 widened, DOUBLE as raw bits
        C.cnull[k] = is_null ? 1 : 0;
    }
    for (int i = threadIdx.x; i < C.ncalls; i += blockDim.x) C.cstate[i] = C.last[i];
}

}  // namespace

struct gsql_window {
    gsql_ctx *ctx;
    gsql_window_spec spec;
    int32_t out_types[GSQL_MAX_AGGS];  // one per call
    int32_t in_type[GSQL_MAX_AGGS];
    bool has_carry = false;
    DevBuf ckey, cnull, cstate, last;
};

extern "C" gsql_status gsql_window_create(gsql_ctx *ctx, const gsql_window_spec *spec, gsql_window **out) {
    if (!ctx || !spec || !out) return GSQL_E_INVALID;
    if (ctx->sticky) return GSQL_E_CUDA;
    *out = nullptr;
    const gsql_window_spec &s = *spec;
    if (s.n_input_cols < 0 || s.n_input_cols > GSQL_MAX_COLS || s.npart < 0 || s.npart > GSQL_MAX_KEYS || s.ncalls < 1 ||
        s.ncalls > GSQL_MAX_AGGS)
        return gsql_set_error(ctx, GSQL_E_INVALID, "window: bad spec sizes");
    for (int i = 0; i < s.n_input_cols; i++) {
        if (s.input_types[i] == GSQL_T_DEC128) return gsql_set_error(ctx, GSQL_E_UNSUPPORTED, "window: input col %d is DEC128", i);
        if (s.input_types[i] < GSQL_T_INT32 || s.input_types[i] > GSQL_T_FP64) return gsql_set_error(ctx, GSQL_E_INVALID, "window: input col %d type", i);
    }
    for (int k = 0; k < s.npart; k++)
        if (s.part_cols[k] < 0 || s.part_cols[k] >= s.n_input_cols) return gsql_set_error(ctx, GSQL_E_INVALID, "window: partition col out of range");
    int32_t out_types[GSQL_MAX_AGGS], in_type[GSQL_MAX_AGGS];
    for (int i = 0; i < s.ncalls; i++) {
        const gsql_agg_call &c = s.calls[i];
        // NonFrameOverWindowExec calls Aggregator.accumulate directly, so the stock operator ignores FILTER: refused
        if (c.filter_arg >= 0) return gsql_set_error(ctx, GSQL_E_UNSUPPORTED, "window: call %d has a FILTER argument", i);
        const bool rank = c.kind == GSQL_AGG_RANK || c.kind == GSQL_AGG_DENSE_RANK;
        const bool known = c.kind == GSQL_AGG_ROW_NUMBER || rank || (c.kind >= GSQL_AGG_COUNT_STAR && c.kind <= GSQL_AGG_SUM0);
        if (!known) return gsql_set_error(ctx, GSQL_E_UNSUPPORTED, "window: call %d: kind %d", i, c.kind);
        if (rank && c.ncols > 4) return gsql_set_error(ctx, GSQL_E_UNSUPPORTED, "window: call %d: more than 4 peer columns", i);
        int lo = 1, hi = 1;
        if (c.kind == GSQL_AGG_ROW_NUMBER || c.kind == GSQL_AGG_COUNT_STAR) lo = hi = 0;
        else if (rank) lo = 0, hi = 4;
        else if (c.kind == GSQL_AGG_COUNT) hi = 4;
        if (c.ncols < lo || c.ncols > hi) return gsql_set_error(ctx, GSQL_E_INVALID, "window: call %d: argument count", i);
        for (int q = 0; q < c.ncols; q++)
            if (c.cols[q] < 0 || c.cols[q] >= s.n_input_cols) return gsql_set_error(ctx, GSQL_E_INVALID, "window: call %d: column out of range", i);
        in_type[i] = c.ncols > 0 && !rank ? s.input_types[c.cols[0]] : GSQL_T_INT64;
        if (c.kind == GSQL_AGG_AVG && in_type[i] != GSQL_T_FP64) return gsql_set_error(ctx, GSQL_E_UNSUPPORTED, "window: AVG(integer) -> DECIMAL");
        if (c.kind == GSQL_AGG_SUM0 && in_type[i] != GSQL_T_INT64) return gsql_set_error(ctx, GSQL_E_UNSUPPORTED, "window: SUM0 needs BIGINT input");
        out_types[i] = (c.kind == GSQL_AGG_ROW_NUMBER || rank) ? GSQL_T_INT64 : agg_out_type(c.kind, in_type[i]);
    }
    gsql_window *w = new gsql_window();
    w->ctx = ctx;
    gsql_ctx_retain(ctx);
    w->spec = s;
    memcpy(w->out_types, out_types, sizeof(out_types));
    memcpy(w->in_type, in_type, sizeof(in_type));
    cudaSetDevice(ctx->device);
    gsql_status st = w->ckey.alloc(ctx, WT_CARRY_KEYS * 8);
    if (st == GSQL_OK) st = w->cnull.alloc(ctx, WT_CARRY_KEYS);
    if (st == GSQL_OK) st = w->cstate.alloc(ctx, GSQL_MAX_AGGS * sizeof(SState));
    if (st == GSQL_OK) st = w->last.alloc(ctx, GSQL_MAX_AGGS * sizeof(SState));
    if (st != GSQL_OK) {
        delete w;
        gsql_ctx_release(ctx);
        return st;
    }
    *out = w;
    return GSQL_OK;
}

extern "C" void gsql_window_destroy(gsql_window *w) {
    if (!w) return;
    gsql_ctx *ctx = w->ctx;
    cudaSetDevice(ctx->device);
    delete w;
    if (!ctx->sticky) cudaStreamSynchronize(ctx->stream);  // frees are stream-ordered: return the memory before returning
    gsql_ctx_release(ctx);
}

extern "C" gsql_status gsql_window_output_schema(gsql_window *w, int32_t *ncols, int32_t *types) {
    if (!w || !ncols) return GSQL_E_INVALID;
    const gsql_window_spec &s = w->spec;
    *ncols = s.n_input_cols + s.ncalls;
    if (types) {
        for (int i = 0; i < s.n_input_cols; i++) types[i] = s.input_types[i];
        for (int i = 0; i < s.ncalls; i++) types[s.n_input_cols + i] = w->out_types[i];
    }
    return GSQL_OK;
}

extern "C" gsql_status gsql_window_apply(gsql_window *w, const gsql_batch *in, gsql_batch *out) {
    if (!w || !in || !out) return GSQL_E_INVALID;
    gsql_ctx *ctx = w->ctx;
    if (ctx->sticky) return GSQL_E_CUDA;
    const gsql_window_spec &s = w->spec;
    GSQL_TRY(validate_batch(ctx, in, s.n_input_cols, s.input_types));
    GSQL_TRY(validate_batch(ctx, out, s.ncalls, w->out_types));
    for (int c = 0; c < s.ncalls; c++) {
        if (!out->cols[c].nulls) return gsql_set_error(ctx, GSQL_E_INVALID, "window output column %d needs a nulls buffer", c);
        // values are stored as whole 4- or 8-byte words (DEC128 as two 8-byte words)
        const uintptr_t align = w->out_types[c] == GSQL_T_INT32 ? 4 : 8;
        if (out->mem == GSQL_MEM_DEVICE && (reinterpret_cast<uintptr_t>(out->cols[c].data) & (align - 1)) != 0)
            return gsql_set_error(ctx, GSQL_E_INVALID, "window output column %d is not aligned to its element", c);
    }
    const int64_t n = in->rows;
    if (n > ((int64_t)1 << 40)) return gsql_set_error(ctx, GSQL_E_CAPACITY, "window: batch of %lld rows is too large", (long long)n);
    out->rows = n;
    if (n == 0) return GSQL_OK;
    GSQL_CUDA(ctx, cudaSetDevice(ctx->device));
    const int ntiles = (int)div_up(n, WT_TILE);
    StagedBatch sb;
    GSQL_TRY(stage_batch(ctx, in, &sb));

    WinParams P;
    memset(&P, 0, sizeof(P));
    P.in.n = sb.ncols;
    for (int c = 0; c < sb.ncols; c++) P.in.c[c] = sb.cols[c];
    P.rows = n;
    P.ntiles = ntiles;
    P.ncalls = s.ncalls;
    P.npart = s.npart;
    P.reset = s.reset_each_row ? 1 : 0;
    P.has_carry = w->has_carry ? 1 : 0;
    for (int k = 0; k < s.npart; k++) P.part_col[k] = s.part_cols[k];
    DevBuf host_out[GSQL_MAX_AGGS], host_nulls[GSQL_MAX_AGGS];  // device staging of a host `out`
    DevBuf tile_buf[GSQL_MAX_AGGS];
    for (int i = 0; i < s.ncalls; i++) {
        const gsql_agg_call &c = s.calls[i];
        WinCall &cl = P.call[i];
        cl.kind = c.kind;
        cl.in_type = w->in_type[i];
        cl.out_type = w->out_types[i];
        cl.ncols = c.ncols;
        for (int q = 0; q < 4; q++) cl.cols[q] = q < c.ncols ? c.cols[q] : 0;
        if (out->mem == GSQL_MEM_DEVICE) {
            P.out[i].data = out->cols[i].data;
            P.out[i].nulls = out->cols[i].nulls;
        } else {
            GSQL_TRY(host_out[i].alloc(ctx, (size_t)n * gsql_type_width(w->out_types[i])));
            GSQL_TRY(host_nulls[i].alloc(ctx, (size_t)n));
            P.out[i].data = host_out[i].p;
            P.out[i].nulls = host_nulls[i].as<uint8_t>();
        }
        size_t tile_bytes = 0;
        GSQL_CUDA(ctx, P.tiles[i].AllocationSize(ntiles, tile_bytes));
        GSQL_TRY(tile_buf[i].alloc(ctx, tile_bytes));
        GSQL_CUDA(ctx, P.tiles[i].Init(ntiles, tile_buf[i].p, tile_bytes));
    }
    P.ckey = w->ckey.as<int64_t>();
    P.cnull = w->cnull.as<uint8_t>();
    P.cstate = w->cstate.as<SState>();
    P.last = w->last.as<SState>();
    {
        KernelScope ks(ctx, "win_init");
        k_win_init<<<(int)div_up(ntiles + 32, 256), 256, 0, ctx->stream>>>(P);
    }
    GSQL_CUDA(ctx, cudaGetLastError());
    {
        KernelScope ks(ctx, "win_tile");
        k_win_tile<<<ntiles, WT_THREADS, 0, ctx->stream>>>(P);
    }
    GSQL_CUDA(ctx, cudaGetLastError());

    WinCarry C;
    memset(&C, 0, sizeof(C));
    C.in = P.in;
    C.row = n - 1;
    C.ncalls = s.ncalls;
    C.nkeys = WT_CARRY_KEYS;
    for (int k = 0; k < WT_CARRY_KEYS; k++) C.key_col[k] = -1;
    for (int k = 0; k < s.npart; k++) C.key_col[k] = s.part_cols[k];
    for (int i = 0; i < s.ncalls; i++)
        if (s.calls[i].kind == GSQL_AGG_RANK || s.calls[i].kind == GSQL_AGG_DENSE_RANK)
            for (int q = 0; q < s.calls[i].ncols; q++) C.key_col[GSQL_MAX_KEYS + 4 * i + q] = s.calls[i].cols[q];
    C.ckey = w->ckey.as<int64_t>();
    C.cnull = w->cnull.as<uint8_t>();
    C.cstate = w->cstate.as<SState>();
    C.last = w->last.as<SState>();
    {
        KernelScope ks(ctx, "win_carry");
        k_win_carry<<<1, 32, 0, ctx->stream>>>(C);
    }
    GSQL_CUDA(ctx, cudaGetLastError());
    w->has_carry = true;

    if (out->mem == GSQL_MEM_HOST) {
        for (int i = 0; i < s.ncalls; i++) {
            GSQL_CUDA(ctx, cudaMemcpyAsync(out->cols[i].data, host_out[i].p, (size_t)n * gsql_type_width(w->out_types[i]), cudaMemcpyDeviceToHost, ctx->stream));
            GSQL_CUDA(ctx, cudaMemcpyAsync(out->cols[i].nulls, host_nulls[i].p, (size_t)n, cudaMemcpyDeviceToHost, ctx->stream));
        }
    }
    if (in->mem == GSQL_MEM_HOST || out->mem == GSQL_MEM_HOST) GSQL_CUDA(ctx, cudaStreamSynchronize(ctx->stream));
    return GSQL_OK;
}
