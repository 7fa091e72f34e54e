// agg_sorted.cuh — GPU SortAggExec behind gsql_sortagg_* (included at the end of agg.cu; reuses its AggDev state
// arrays, init_value, dbl_sortable, agg_out_type, k_agg_finalize and the spec check agg_check_spec).
//
// Reference path replaced (EX/ = polardbx-executor/src/main/java/com/alibaba/polardbx/executor/):
//   EX/operator/SortAggExec.java:72-112 (doNextChunk), :114-124 (buildRow), :126-135 (checkKeyEqual)
//   EX/mpp/operator/factory/SortAggExecFactory.java (one executor per driver)
//
// A group is a maximal run of adjacent rows whose keys compare equal under NumberType.compare: two NULLs are equal,
// NULL differs from every value, integers by value, doubles by Double.compare (-0.0 and +0.0 differ, every NaN equals
// every NaN).  Unsorted input is not an error: each run is a group.  The key written is the run's first row's, bit for bit.
//
// One batch is one segmented reduction, in two kernels:
//   k_sagg_tile   one CTA per tile of SA_TILE rows, SA_IPT consecutive rows per thread.  Head flags compare each row with
//                 its predecessor (row 0 of a batch with the open group's key); a block scan of the flags plus a decoupled
//                 look-back over the tiles' head counts gives every row its dense group id, without a separate pass over
//                 the keys.  Per aggregate, each thread folds its rows; a block-wide segmented scan over the threads'
//                 partials completes every segment that starts in the tile, which is stored whole (plain stores) at its
//                 group id.  A tile whose first row is not a head publishes that segment's partial as its continuation.
//   k_sagg_fixup  folds the continuations into their groups: one atomic per continuing tile per aggregate.
// No per-row atomics, no grid-wide barrier.  Group ids of a batch are local: slot 0 holds the group left open by the previous
// batch (its key and partial states, carried in by k_sagg_carry), slot g >= 1 the g-th run that starts in the batch.  All
// complete groups are finalised (k_agg_finalize) into the output buffer at once; the last group is carried to the next batch.
#include <cub/agent/single_pass_scan_operators.cuh>
#include <cub/block/block_scan.cuh>

namespace {

constexpr int SA_THREADS = 256, SA_IPT = 8, SA_TILE = SA_THREADS * SA_IPT;

struct SState {  // one aggregate's partial over a run of rows; also the segmented-scan element
    long long l;   // AggDev::l
    long long x;   // AggDev::hi (SUM of integers) or the bits of AggDev::d (floating sums)
    int has;       // AggDev::has
    int f;         // scan only: a run starts in the rows this partial covers
};
__device__ __forceinline__ double sa_d(const SState &s) { return __longlong_as_double(s.x); }
__device__ __forceinline__ void sa_set_d(SState &s, double d) { s.x = __double_as_longlong(d); }

struct SaggParams {
    DColSet in;
    int32_t nkeys, naggs, has_open, pad;
    int64_t rows;
    int32_t ntiles, pad2;
    int32_t keycol[GSQL_MAX_KEYS];
    int64_t *gkey[GSQL_MAX_KEYS];  // group keys by local group id: INT widened to 64 bits, DOUBLE as raw bits
    uint8_t *gnull[GSQL_MAX_KEYS];
    AggDev agg[GSQL_MAX_AGGS];
    SState *cont;                  // [naggs][ntiles]: the partial of the segment a tile continues
    int64_t *cont_gid;             // [ntiles]: its group id; -1 when the tile's first row starts a group
    unsigned long long *total;     // number of groups that start in the batch
    cub::ScanTileState<long long> tiles;
};

__device__ __forceinline__ bool sa_key_eq(const KeyVal &a, const KeyVal &b, int t) {
    if (a.is_null || b.is_null) return a.is_null == b.is_null;
    if (t == GSQL_T_FP64) return gsql_double_bits(__longlong_as_double(a.i)) == gsql_double_bits(__longlong_as_double(b.i));
    return a.i == b.i;
}

__device__ __forceinline__ SState sa_zero(int kind) {
    SState s;
    s.l = init_value(kind);
    s.x = 0;  // 128-bit high word 0, or +0.0
    s.has = 0;
    s.f = 0;
    return s;
}

__device__ __forceinline__ void sa_add128(SState &s, long long v) {
    unsigned long long lo = (unsigned long long)s.l + (unsigned long long)v;
    s.x += (lo < (unsigned long long)s.l ? 1 : 0) + (v < 0 ? -1 : 0);
    s.l = (long long)lo;
}

// Folds row r into s: accumulate()'s rules, without the atomics.
__device__ __forceinline__ void sa_add(const DColSet &in, const AggDev &a, SState &s, int64_t r) {
    switch (a.kind) {
    case GSQL_AGG_COUNT_STAR: s.l++; return;
    case GSQL_AGG_COUNT:
        for (int i = 0; i < a.ncols; i++)
            if (in_null(in.c[a.cols[i]], r)) return;
        s.l++;
        return;
    default: break;
    }
    const DCol &c = in.c[a.cols[0]];
    if (in_null(c, r)) return;
    switch (a.kind) {
    case GSQL_AGG_SUM:
        if (a.in_type == GSQL_T_FP64) {
            double x = in_f64(c, r);
            sa_set_d(s, s.has ? sa_d(s) + x : x);
        } else {
            sa_add128(s, in_i64(c, r));
        }
        s.has = 1;
        return;
    case GSQL_AGG_AVG: {
        double x = in_f64(c, r);
        sa_set_d(s, s.has ? sa_d(s) + x : x);
        s.l++;
        s.has = 1;
        return;
    }
    case GSQL_AGG_SUM0: s.l = (long long)((unsigned long long)s.l + (unsigned long long)in_i64(c, r)); return;
    case GSQL_AGG_AVG_MERGE: {
        double x = in_f64(c, r);
        sa_set_d(s, s.has ? sa_d(s) + x : x);
        s.has = 1;
        const DCol &n = in.c[a.cols[1]];
        if (!in_null(n, r)) s.l = (long long)((unsigned long long)s.l + (unsigned long long)in_i64(n, r));
        return;
    }
    default: {  // MIN / MAX on the order-preserving image
        bool mx = a.kind == GSQL_AGG_MAX;
        long long v = a.in_type == GSQL_T_FP64 ? dbl_sortable(in_f64(c, r), mx) : in_i64(c, r);
        s.l = mx ? (v > s.l ? v : s.l) : (v < s.l ? v : s.l);
        s.has = 1;
    }
    }
}

// a then b (b's rows follow a's)
__device__ __forceinline__ SState sa_combine(int kind, int in_type, const SState &a, const SState &b) {
    SState s = a;
    s.has = a.has | b.has;
    switch (kind) {
    case GSQL_AGG_COUNT_STAR: case GSQL_AGG_COUNT: case GSQL_AGG_SUM0:
        s.l = (long long)((unsigned long long)a.l + (unsigned long long)b.l);
        break;
    case GSQL_AGG_SUM:
        if (in_type == GSQL_T_FP64) {
            s.x = a.has ? (b.has ? __double_as_longlong(sa_d(a) + sa_d(b)) : a.x) : b.x;
        } else {
            unsigned long long lo = (unsigned long long)a.l + (unsigned long long)b.l;
            s.x = a.x + b.x + (lo < (unsigned long long)a.l ? 1 : 0);
            s.l = (long long)lo;
        }
        break;
    case GSQL_AGG_AVG: case GSQL_AGG_AVG_MERGE:
        s.x = a.has ? (b.has ? __double_as_longlong(sa_d(a) + sa_d(b)) : a.x) : b.x;
        s.l = (long long)((unsigned long long)a.l + (unsigned long long)b.l);
        break;
    case GSQL_AGG_MAX: s.l = b.l > a.l ? b.l : a.l; break;
    default: s.l = b.l < a.l ? b.l : a.l; break;  // MIN
    }
    return s;
}

struct SaSegOp {  // reduce-by-segment: a run that starts in b discards a
    int kind, in_type;
    __device__ __forceinline__ SState operator()(const SState &a, const SState &b) const {
        SState o = b.f ? b : sa_combine(kind, in_type, a, b);
        o.f = a.f | b.f;
        return o;
    }
};

__device__ __forceinline__ void sa_store(const AggDev &a, int64_t g, const SState &s) {
    a.l[g] = s.l;
    if (a.hi) a.hi[g] = s.x;
    if (a.d) a.d[g] = sa_d(s);
    a.has[g] = (uint8_t)s.has;
}

__global__ void k_sagg_init(cub::ScanTileState<long long> tiles, int ntiles) { tiles.InitializeStatus(ntiles); }

__global__ void __launch_bounds__(SA_THREADS, 2) k_sagg_tile(const __grid_constant__ SaggParams P) {
    typedef cub::BlockScan<long long, SA_THREADS> CountScan;
    typedef cub::TilePrefixCallbackOp<long long, ::cuda::std::plus<long long>, cub::ScanTileState<long long>> LookBack;
    typedef cub::BlockScan<SState, SA_THREADS> SegScan;
    __shared__ struct {
        typename CountScan::TempStorage count;
        typename LookBack::TempStorage lookback;
        typename SegScan::TempStorage seg;
        long long tile_base;
    } sm;

    const int tile = blockIdx.x;
    const int64_t t0 = (int64_t)tile * SA_TILE;
    const int64_t r0 = t0 + (int64_t)threadIdx.x * SA_IPT;
    const int nlive = P.rows - r0 >= SA_IPT ? SA_IPT : (P.rows > r0 ? (int)(P.rows - r0) : 0);
    const unsigned live_mask = nlive == 32 ? ~0u : ((1u << nlive) - 1);

    // ---- head flags: bit i = row r0 + i starts a group
    unsigned same = live_mask;
    if (r0 == 0 && !P.has_open) same &= ~1u;
#pragma unroll 1
    for (int k = 0; k < P.nkeys; k++) {
        const DCol &c = P.in.c[P.keycol[k]];
        const int t = c.type;
        KeyVal prev;
        if (nlive == 0) break;
        if (r0 == 0) {
            prev.i = P.gkey[k][0];
            prev.is_null = P.gnull[k][0] != 0;
        } else {
            prev = gsql_load_key(c, r0 - 1, t);
        }
#pragma unroll
        for (int i = 0; i < SA_IPT; i++) {
            if (i < nlive) {
                KeyVal v = gsql_load_key(c, r0 + i, t);
                if (!sa_key_eq(v, prev, t)) same &= ~(1u << i);
                prev = v;
            }
        }
    }
    const unsigned heads = ~same & live_mask;

    // ---- dense group ids: block scan of the head counts, decoupled look-back over the tiles
    long long excl;
    cub::ScanTileState<long long> ts = P.tiles;
    if (tile == 0) {
        long long block_total;
        CountScan(sm.count).ExclusiveSum((long long)__popc(heads), excl, block_total);
        if (threadIdx.x == 0) ts.SetInclusive(0, block_total);
    } else {
        LookBack prefix(ts, sm.lookback, ::cuda::std::plus<long long>(), tile);
        CountScan(sm.count).ExclusiveSum((long long)__popc(heads), excl, prefix);
    }
    if (threadIdx.x == 0) sm.tile_base = excl;
    if (tile == P.ntiles - 1 && threadIdx.x == SA_THREADS - 1) *P.total = (unsigned long long)(excl + __popc(heads));
    __syncthreads();
    const long long tile_base = sm.tile_base;  // group id of the tile's first row when it continues a group
    if (threadIdx.x == 0) P.cont_gid[tile] = (heads & 1u) ? -1 : tile_base;

    // keys of the groups that start here: the head row's, bit for bit
#pragma unroll 1
    for (int k = 0; k < P.nkeys; k++) {
        const DCol &c = P.in.c[P.keycol[k]];
        long long g = excl;
        for (int i = 0; i < nlive; i++) {
            if ((heads >> i) & 1u) {
                g++;
                KeyVal v = gsql_load_key(c, r0 + i, c.type);
                P.gkey[k][g] = v.i;
                P.gnull[k][g] = v.is_null ? 1 : 0;
            }
        }
    }

    // ---- per aggregate: thread partials, then a segmented scan over the threads
    const int last_thread = (int)((P.rows - 1 - t0) / SA_IPT < SA_THREADS - 1 ? (P.rows - 1 - t0) / SA_IPT : SA_THREADS - 1);
    const int first_head = heads ? __ffs(heads) - 1 : -1;
#pragma unroll 1
    for (int ai = 0; ai < P.naggs; ai++) {
        const AggDev &a = P.agg[ai];
        SState cur = sa_zero(a.kind), pre = cur;
        bool owned = false;  // `cur` started at a head of this thread
        long long g = excl;  // group id of the current row
        for (int i = 0; i < nlive; i++) {
            if ((heads >> i) & 1u) {
                if (owned) sa_store(a, g, cur);  // a run that starts and ends inside the thread
                else pre = cur;
                cur = sa_zero(a.kind);
                owned = true;
                g++;
            }
            sa_add(P.in, a, cur, r0 + i);
        }
        if (!owned) pre = cur;
        SState mine = cur, ex, id = sa_zero(a.kind);
        mine.f = owned ? 1 : 0;
        SaSegOp op{a.kind, a.in_type};
        __syncthreads();  // the previous aggregate's scan storage is free again
        SegScan(sm.seg).ExclusiveScan(mine, ex, id, op);
        if (owned) {  // the run that this thread's first head closes
            SState closed = sa_combine(a.kind, a.in_type, ex, pre);
            if (ex.f) sa_store(a, excl, closed);  // starts in an earlier thread of this tile
            else if (!(threadIdx.x == 0 && first_head == 0)) P.cont[(int64_t)ai * P.ntiles + tile] = closed;
        }
        if ((int)threadIdx.x == last_thread) {  // the tile's last run
            SState inc = op(ex, mine);
            if (inc.f) sa_store(a, g, inc);
            else P.cont[(int64_t)ai * P.ntiles + tile] = inc;
        }
    }
}

// One thread per tile: folds the tile's continuation into its group (accumulate()'s combine rules).
__global__ void __launch_bounds__(256) k_sagg_fixup(const __grid_constant__ SaggParams P) {
    const int64_t t = blockIdx.x * (int64_t)blockDim.x + threadIdx.x;
    if (t >= P.ntiles) return;
    const int64_t g = P.cont_gid[t];
    if (g < 0) return;
    for (int ai = 0; ai < P.naggs; ai++) {
        const AggDev &a = P.agg[ai];
        const SState b = P.cont[(int64_t)ai * P.ntiles + t];
        switch (a.kind) {
        case GSQL_AGG_COUNT_STAR: case GSQL_AGG_COUNT: case GSQL_AGG_SUM0:
            atomicAdd(reinterpret_cast<unsigned long long *>(&a.l[g]), (unsigned long long)b.l);
            break;
        case GSQL_AGG_SUM:
            if (!b.has) break;
            if (a.in_type == GSQL_T_FP64) {
                atomicAdd(&a.d[g], sa_d(b));
            } else {
                unsigned long long old = atomicAdd(reinterpret_cast<unsigned long long *>(&a.l[g]), (unsigned long long)b.l);
                long long carry = b.x + ((old + (unsigned long long)b.l) < old ? 1 : 0);
                if (carry) atomicAdd(reinterpret_cast<unsigned long long *>(&a.hi[g]), (unsigned long long)carry);
            }
            a.has[g] = 1;
            break;
        case GSQL_AGG_AVG: case GSQL_AGG_AVG_MERGE:
            if (!b.has) break;
            atomicAdd(&a.d[g], sa_d(b));
            atomicAdd(reinterpret_cast<unsigned long long *>(&a.l[g]), (unsigned long long)b.l);
            a.has[g] = 1;
            break;
        case GSQL_AGG_MAX:
            if (!b.has) break;
            atomicMax(reinterpret_cast<long long *>(&a.l[g]), b.l);
            a.has[g] = 1;
            break;
        default:
            if (!b.has) break;
            atomicMin(reinterpret_cast<long long *>(&a.l[g]), b.l);
            a.has[g] = 1;
        }
    }
}

struct SaggCarry {  // group `from` of one set of group arrays -> group 0 of another
    int32_t nkeys, naggs;
    int64_t from;
    const int64_t *skey[GSQL_MAX_KEYS];
    const uint8_t *snull[GSQL_MAX_KEYS];
    int64_t *dkey[GSQL_MAX_KEYS];
    uint8_t *dnull[GSQL_MAX_KEYS];
    AggDev src[GSQL_MAX_AGGS], dst[GSQL_MAX_AGGS];
};

__global__ void k_sagg_carry(const __grid_constant__ SaggCarry C) {
    const int64_t f = C.from;
    for (int k = 0; k < C.nkeys; k++) {
        C.dkey[k][0] = C.skey[k][f];
        C.dnull[k][0] = C.snull[k][f];
    }
    for (int i = 0; i < C.naggs; i++) {
        const AggDev &s = C.src[i], &d = C.dst[i];
        d.l[0] = s.l[f];
        if (s.hi) d.hi[0] = s.hi[f];
        if (s.d) d.d[0] = s.d[f];
        d.has[0] = s.has[f];
    }
}

}  // namespace

// Group keys and aggregate states for `n` groups, by group id.
struct SaggGroups {
    DevBuf gkey[GSQL_MAX_KEYS], gnull[GSQL_MAX_KEYS];
    DevBuf l[GSQL_MAX_AGGS], hi[GSQL_MAX_AGGS], d[GSQL_MAX_AGGS], has[GSQL_MAX_AGGS];
};

struct gsql_sortagg {
    gsql_ctx *ctx;
    gsql_agg_spec spec;
    int32_t nkeys = 0, naggs = 0, nout = 0;
    int32_t in_type[GSQL_MAX_AGGS];
    int32_t out_types[GSQL_MAX_COLS];
    SaggGroups open;        // the group the last batch ended in (group 0), while has_open
    bool has_open = false, finished = false;
    DevBuf out_data[GSQL_MAX_COLS], out_nulls[GSQL_MAX_COLS];  // finalised groups; rows [cursor, out_n) not yet returned
    int64_t out_cap = 0, out_n = 0, cursor = 0;
};

static bool sagg_has_hi(const gsql_sortagg *s, int i) { return s->spec.aggs[i].kind == GSQL_AGG_SUM && s->in_type[i] != GSQL_T_FP64; }
static bool sagg_has_d(const gsql_sortagg *s, int i) {
    int k = s->spec.aggs[i].kind;
    return (k == GSQL_AGG_SUM && s->in_type[i] == GSQL_T_FP64) || k == GSQL_AGG_AVG || k == GSQL_AGG_AVG_MERGE;
}

static gsql_status sagg_alloc_groups(gsql_sortagg *s, SaggGroups *G, int64_t n) {
    for (int k = 0; k < s->nkeys; k++) {
        GSQL_TRY(G->gkey[k].alloc(s->ctx, (size_t)n * 8));
        GSQL_TRY(G->gnull[k].alloc(s->ctx, (size_t)n));
    }
    for (int i = 0; i < s->naggs; i++) {
        GSQL_TRY(G->l[i].alloc(s->ctx, (size_t)n * 8));
        GSQL_TRY(G->has[i].alloc(s->ctx, (size_t)n));
        if (sagg_has_hi(s, i)) GSQL_TRY(G->hi[i].alloc(s->ctx, (size_t)n * 8));
        if (sagg_has_d(s, i)) GSQL_TRY(G->d[i].alloc(s->ctx, (size_t)n * 8));
    }
    return GSQL_OK;
}

static AggDev sagg_dev(const gsql_sortagg *s, const SaggGroups &G, int i) {
    AggDev d;
    memset(&d, 0, sizeof(d));
    const gsql_agg_call &c = s->spec.aggs[i];
    d.kind = c.kind;
    d.in_type = s->in_type[i];
    d.ncols = c.ncols;
    d.filter_col = -1;
    for (int q = 0; q < 4; q++) d.cols[q] = c.cols[q];
    d.l = G.l[i].as<int64_t>();
    d.hi = sagg_has_hi(s, i) ? G.hi[i].as<int64_t>() : nullptr;
    d.d = sagg_has_d(s, i) ? G.d[i].as<double>() : nullptr;
    d.has = G.has[i].as<uint8_t>();
    return d;
}

static gsql_status sagg_carry(gsql_sortagg *s, const SaggGroups &from, int64_t g, SaggGroups &to) {
    SaggCarry C;
    memset(&C, 0, sizeof(C));
    C.nkeys = s->nkeys;
    C.naggs = s->naggs;
    C.from = g;
    for (int k = 0; k < s->nkeys; k++) {
        C.skey[k] = from.gkey[k].as<int64_t>();
        C.snull[k] = from.gnull[k].as<uint8_t>();
        C.dkey[k] = to.gkey[k].as<int64_t>();
        C.dnull[k] = to.gnull[k].as<uint8_t>();
    }
    for (int i = 0; i < s->naggs; i++) {
        C.src[i] = sagg_dev(s, from, i);
        C.dst[i] = sagg_dev(s, to, i);
    }
    if (s->nkeys == 0 && s->naggs == 0) return GSQL_OK;
    KernelScope ks(s->ctx, "sagg_carry");
    k_sagg_carry<<<1, 1, 0, s->ctx->stream>>>(C);
    GSQL_CUDA(s->ctx, cudaGetLastError());
    return GSQL_OK;
}

// Room for m more output rows; rows already returned are dropped, so that what is held stays O(rows not yet returned).
static gsql_status sagg_reserve(gsql_sortagg *s, int64_t m) {
    gsql_ctx *ctx = s->ctx;
    const int64_t live = s->out_n - s->cursor, need = live + m;
    if (live == 0) s->out_n = s->cursor = 0;
    if (s->out_n + m <= s->out_cap && s->out_cap <= 4 * std::max<int64_t>(need, 1024)) return GSQL_OK;
    const int64_t ncap = std::max<int64_t>(2 * need, 1024);
    for (int c = 0; c < s->nout; c++) {
        const int w = gsql_type_width(s->out_types[c]);
        DevBuf nd, nn;
        GSQL_TRY(nd.alloc(ctx, (size_t)ncap * w));
        GSQL_TRY(nn.alloc(ctx, (size_t)ncap));
        if (live) {
            GSQL_CUDA(ctx, cudaMemcpyAsync(nd.p, (char *)s->out_data[c].p + (size_t)s->cursor * w, (size_t)live * w, cudaMemcpyDeviceToDevice, ctx->stream));
            GSQL_CUDA(ctx, cudaMemcpyAsync(nn.p, (char *)s->out_nulls[c].p + s->cursor, (size_t)live, cudaMemcpyDeviceToDevice, ctx->stream));
        }
        std::swap(s->out_data[c].p, nd.p);
        std::swap(s->out_data[c].bytes, nd.bytes);
        s->out_data[c].ctx = ctx;
        std::swap(s->out_nulls[c].p, nn.p);
        std::swap(s->out_nulls[c].bytes, nn.bytes);
        s->out_nulls[c].ctx = ctx;
    }
    s->out_cap = ncap;
    s->out_n = live;
    s->cursor = 0;
    return GSQL_OK;
}

// Appends groups [g0, g0 + m) of G, finalised (writeResultTo), to the output rows.
static gsql_status sagg_emit(gsql_sortagg *s, const SaggGroups &G, int64_t g0, int64_t m) {
    if (m <= 0) return GSQL_OK;
    GSQL_TRY(sagg_reserve(s, m));
    FinalParams F;
    memset(&F, 0, sizeof(F));
    F.nkeys = s->nkeys;
    F.naggs = s->naggs;
    F.ngroups = m;
    for (int k = 0; k < s->nkeys; k++) {
        F.gkey[k] = G.gkey[k].as<int64_t>() + g0;
        F.gnull[k] = G.gnull[k].as<uint8_t>() + g0;
        F.key_types[k] = s->out_types[k];
    }
    for (int i = 0; i < s->naggs; i++) {
        AggDev d = sagg_dev(s, G, i);
        d.l += g0;
        if (d.hi) d.hi += g0;
        if (d.d) d.d += g0;
        d.has += g0;
        F.agg[i] = d;
    }
    for (int c = 0; c < s->nout; c++) {
        F.out[c].data = (char *)s->out_data[c].p + (size_t)s->out_n * gsql_type_width(s->out_types[c]);
        F.out[c].nulls = s->out_nulls[c].as<uint8_t>() + s->out_n;
        F.out[c].type = s->out_types[c];
    }
    if (s->nout > 0) {
        KernelScope ks(s->ctx, "sagg_finalize");
        k_agg_finalize<<<grid_rows(s->ctx, m, 256, 8), 256, 0, s->ctx->stream>>>(F);
    }
    GSQL_CUDA(s->ctx, cudaGetLastError());
    s->out_n += m;
    return GSQL_OK;
}

extern "C" gsql_status gsql_sortagg_create(gsql_ctx *ctx, const gsql_agg_spec *spec, gsql_sortagg **out) {
    if (!ctx || !spec || !out) return GSQL_E_INVALID;
    if (ctx->sticky) return GSQL_E_CUDA;
    *out = nullptr;
    const gsql_agg_spec &sp = *spec;
    int32_t in_type[GSQL_MAX_AGGS], out_types[GSQL_MAX_COLS], nout = 0;
    GSQL_TRY(agg_check_spec(ctx, sp, in_type, out_types, &nout));
    // The fused scan-side Project / Filter of the hash aggregation has no SortAgg plan shape.  FILTER clauses are refused:
    // the stock SortAggExec calls Aggregator.accumulate directly (SortAggExec.java:92-101) and so ignores filterArg, which only
    // AggOpenHashMap.putChunk applies; refusing keeps such plans on the stock operator instead of silently diverging from it.
    if (sp.n_derived != 0) return gsql_set_error(ctx, GSQL_E_UNSUPPORTED, "sortagg: derived columns are not supported");
    if (sp.row_filter_op != GSQL_CMP_NONE) return gsql_set_error(ctx, GSQL_E_UNSUPPORTED, "sortagg: a row filter is not supported");
    for (int i = 0; i < sp.naggs; i++)
        if (sp.aggs[i].filter_arg >= 0) return gsql_set_error(ctx, GSQL_E_UNSUPPORTED, "sortagg: agg %d has a FILTER argument", i);
    gsql_sortagg *s = new gsql_sortagg();
    s->ctx = ctx;
    gsql_ctx_retain(ctx);
    s->spec = sp;
    s->nkeys = sp.ngroups;
    s->naggs = sp.naggs;
    s->nout = nout;
    memcpy(s->in_type, in_type, sizeof(in_type));
    memcpy(s->out_types, out_types, sizeof(out_types));
    cudaSetDevice(ctx->device);
    gsql_status st = sagg_alloc_groups(s, &s->open, 1);
    if (st != GSQL_OK) {
        delete s;
        gsql_ctx_release(ctx);
        return st;
    }
    *out = s;
    return GSQL_OK;
}

extern "C" void gsql_sortagg_destroy(gsql_sortagg *s) {
    if (!s) return;
    gsql_ctx *ctx = s->ctx;
    cudaSetDevice(ctx->device);
    delete s;
    if (!ctx->sticky) cudaStreamSynchronize(ctx->stream);  // frees are stream-ordered: return the memory before returning
    gsql_ctx_release(ctx);
}

extern "C" gsql_status gsql_sortagg_consume(gsql_sortagg *s, const gsql_batch *batch, int64_t *ready) {
    if (!s) return GSQL_E_INVALID;
    gsql_ctx *ctx = s->ctx;
    if (ctx->sticky) return GSQL_E_CUDA;
    if (s->finished) return gsql_set_error(ctx, GSQL_E_STATE, "consume after finish");
    GSQL_TRY(validate_batch(ctx, batch, s->spec.n_input_cols, s->spec.input_types));
    if (batch->rows > 0) {
        GSQL_CUDA(ctx, cudaSetDevice(ctx->device));
        const int64_t n = batch->rows;
        if (div_up(n, SA_TILE) > 0x7fffffff) return gsql_set_error(ctx, GSQL_E_CAPACITY, "sortagg: batch of %lld rows is too large", (long long)n);
        const int ntiles = (int)div_up(n, SA_TILE);
        StagedBatch sb;
        GSQL_TRY(stage_batch(ctx, batch, &sb));
        SaggGroups G;  // group 0 = the open group, then one per run that starts in the batch
        GSQL_TRY(sagg_alloc_groups(s, &G, n + 1));
        if (s->has_open) GSQL_TRY(sagg_carry(s, s->open, 0, G));
        size_t tile_bytes = 0;
        cub::ScanTileState<long long> tiles;
        GSQL_CUDA(ctx, tiles.AllocationSize(ntiles, tile_bytes));
        DevBuf tile_buf, cont, cont_gid, total;
        GSQL_TRY(tile_buf.alloc(ctx, tile_bytes));
        GSQL_CUDA(ctx, tiles.Init(ntiles, tile_buf.p, tile_bytes));
        GSQL_TRY(cont.alloc(ctx, (size_t)std::max(s->naggs, 1) * ntiles * sizeof(SState)));
        GSQL_TRY(cont_gid.alloc(ctx, (size_t)ntiles * 8));
        GSQL_TRY(total.alloc(ctx, 8));
        SaggParams P;
        memset(&P, 0, sizeof(P));
        P.in.n = sb.ncols;
        for (int c = 0; c < sb.ncols; c++) P.in.c[c] = sb.cols[c];
        P.nkeys = s->nkeys;
        P.naggs = s->naggs;
        P.has_open = s->has_open ? 1 : 0;
        P.rows = n;
        P.ntiles = ntiles;
        for (int k = 0; k < s->nkeys; k++) {
            P.keycol[k] = s->spec.groups[k];
            P.gkey[k] = G.gkey[k].as<int64_t>();
            P.gnull[k] = G.gnull[k].as<uint8_t>();
        }
        for (int i = 0; i < s->naggs; i++) P.agg[i] = sagg_dev(s, G, i);
        P.cont = cont.as<SState>();
        P.cont_gid = cont_gid.as<int64_t>();
        P.total = total.as<unsigned long long>();
        P.tiles = tiles;
        {
            KernelScope ks(ctx, "sagg_init");
            k_sagg_init<<<(int)div_up(ntiles + 32, 256), 256, 0, ctx->stream>>>(tiles, ntiles);
        }
        GSQL_CUDA(ctx, cudaGetLastError());
        {
            KernelScope ks(ctx, "sagg_tile");
            k_sagg_tile<<<ntiles, SA_THREADS, 0, ctx->stream>>>(P);
        }
        GSQL_CUDA(ctx, cudaGetLastError());
        if (s->naggs > 0) {
            KernelScope ks(ctx, "sagg_fixup");
            k_sagg_fixup<<<(int)div_up(ntiles, 256), 256, 0, ctx->stream>>>(P);
        }
        GSQL_CUDA(ctx, cudaGetLastError());
        unsigned long long heads = 0;
        GSQL_CUDA(ctx, cudaMemcpyAsync(&heads, total.p, 8, cudaMemcpyDeviceToHost, ctx->stream));
        GSQL_CUDA(ctx, cudaStreamSynchronize(ctx->stream));
        // groups [first, heads) are complete; group `heads` stays open
        const int64_t first = s->has_open ? 0 : 1;
        GSQL_TRY(sagg_emit(s, G, first, (int64_t)heads - first));
        GSQL_TRY(sagg_carry(s, G, (int64_t)heads, s->open));
        s->has_open = true;
        if (batch->mem == GSQL_MEM_HOST) GSQL_CUDA(ctx, cudaStreamSynchronize(ctx->stream));
    }
    if (ready) *ready = s->out_n - s->cursor;
    return GSQL_OK;
}

extern "C" gsql_status gsql_sortagg_finish(gsql_sortagg *s, int64_t *ready) {
    if (!s) return GSQL_E_INVALID;
    gsql_ctx *ctx = s->ctx;
    if (ctx->sticky) return GSQL_E_CUDA;
    GSQL_CUDA(ctx, cudaSetDevice(ctx->device));
    if (!s->finished) {
        if (s->has_open) GSQL_TRY(sagg_emit(s, s->open, 0, 1));
        s->has_open = false;
        s->finished = true;
    }
    if (ready) *ready = s->out_n - s->cursor;
    return GSQL_OK;
}

extern "C" gsql_status gsql_sortagg_output_schema(gsql_sortagg *s, int32_t *ncols, int32_t *types) {
    if (!s || !ncols) return GSQL_E_INVALID;
    *ncols = s->nout;
    if (types)
        for (int i = 0; i < s->nout; i++) types[i] = s->out_types[i];
    return GSQL_OK;
}

extern "C" gsql_status gsql_sortagg_next(gsql_sortagg *s, gsql_batch *out, int64_t max_rows, int64_t *out_rows) {
    if (!s || !out || !out_rows) return GSQL_E_INVALID;
    gsql_ctx *ctx = s->ctx;
    if (ctx->sticky) return GSQL_E_CUDA;
    GSQL_TRY(validate_batch(ctx, out, s->nout, s->out_types));
    for (int c = 0; c < s->nout; c++)
        if (!out->cols[c].nulls) return gsql_set_error(ctx, GSQL_E_INVALID, "sortagg output column %d needs a nulls buffer", c);
    GSQL_CUDA(ctx, cudaSetDevice(ctx->device));
    int64_t n = s->out_n - s->cursor;
    if (n > max_rows) n = max_rows;
    if (n < 0) n = 0;
    *out_rows = n;
    out->rows = n;
    if (n == 0) return GSQL_OK;
    cudaMemcpyKind kind = out->mem == GSQL_MEM_DEVICE ? cudaMemcpyDeviceToDevice : cudaMemcpyDeviceToHost;
    for (int c = 0; c < s->nout; c++) {
        int w = gsql_type_width(s->out_types[c]);
        GSQL_CUDA(ctx, cudaMemcpyAsync(out->cols[c].data, (char *)s->out_data[c].p + (size_t)s->cursor * w, (size_t)n * w, kind, ctx->stream));
        GSQL_CUDA(ctx, cudaMemcpyAsync(out->cols[c].nulls, (char *)s->out_nulls[c].p + s->cursor, (size_t)n, kind, ctx->stream));
    }
    if (out->mem == GSQL_MEM_HOST) GSQL_CUDA(ctx, cudaStreamSynchronize(ctx->stream));
    s->cursor += n;
    return GSQL_OK;
}
