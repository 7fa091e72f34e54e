// agg_sets.cuh — grouping sets behind gsql_gsagg_* (a HashAgg over an Expand, without materialising the Expand).
// Included by agg.cu: it reuses gsql_agg whole for every set, and the group table's find_group_kv for the merge.
//
// Reference path replaced (EX/ = polardbx-executor/src/main/java/com/alibaba/polardbx/executor/):
//   EX/operator/ExpandExec.java:48-69 (one output chunk per projection per input chunk) feeding
//   EX/operator/HashAggExec.java:133-162 grouped by (all keys, $e), as GroupingSetsToExpandRule.java:255-300 plans it.
//
// Set s references the group columns whose projection is an input column.  Set t derives from set s when every group
// column t references has the same reference in s (ties between equal sets: the later derives from the earlier).  The
// sets that derive from none are roots: each is a gsql_agg over the input, keyed by its referenced columns, with its own
// table, growth and front-end choice.  At finish every other set is built, finest first, from the finished groups of the
// superset with the fewest groups: k_agg_derive reads each parent group's key images and states and merges them into the
// child's table, which is sized from the parent's group count and so never grows.  The group counts of a CUBE lattice
// fall towards the grand total, so the coarse sets cost passes over groups, not over rows.

// The parent's finished groups, as k_agg_derive reads them: key images in the child's key order, and every state.
struct DeriveSrc {
    int64_t ngroups;
    const int64_t *gkey[GSQL_MAX_KEYS];
    const uint8_t *gnull[GSQL_MAX_KEYS];
    AggDev agg[GSQL_MAX_AGGS];
};

// The states of one parent group, folded across the lanes of a warp whose groups land in the same child group.
struct DeriveVal {
    long long l, hi;
    double d;
    bool has;
};

__device__ __forceinline__ DeriveVal derive_load(const AggDev &a, int64_t g, bool live) {
    DeriveVal v{0, 0, 0.0, false};
    if (a.kind == GSQL_AGG_MIN) v.l = 0x7fffffffffffffffLL;  // the identities of atomicMin / atomicMax (init_value)
    if (a.kind == GSQL_AGG_MAX) v.l = (long long)0x8000000000000000ULL;
    if (!live) return v;
    switch (a.kind) {
    case GSQL_AGG_COUNT_STAR: case GSQL_AGG_COUNT: case GSQL_AGG_SUM0:
        v.l = a.l[g];
        return v;
    default: break;
    }
    v.has = a.has[g] != 0;
    if (!v.has) return v;
    switch (a.kind) {
    case GSQL_AGG_SUM:
        if (a.in_type == GSQL_T_FP64) v.d = a.d[g];
        else { v.l = a.l[g]; v.hi = a.hi[g]; }
        break;
    case GSQL_AGG_AVG: v.d = a.d[g]; v.l = a.l[g]; break;
    default: v.l = a.l[g]; break;  // MIN / MAX: the sortable image (FP64) or the integer
    }
    return v;
}

__device__ __forceinline__ void derive_fold(const AggDev &a, DeriveVal &v, const DeriveVal &o) {
    switch (a.kind) {
    case GSQL_AGG_MIN: v.l = o.l < v.l ? o.l : v.l; break;
    case GSQL_AGG_MAX: v.l = o.l > v.l ? o.l : v.l; break;
    case GSQL_AGG_SUM:
        if (a.in_type == GSQL_T_FP64) { v.d += o.d; break; }
        {  // 128-bit (lo, hi) add, carry included
            const unsigned long long lo = (unsigned long long)v.l + (unsigned long long)o.l;
            v.hi = (long long)((unsigned long long)v.hi + (unsigned long long)o.hi + (lo < (unsigned long long)v.l ? 1ULL : 0ULL));
            v.l = (long long)lo;
        }
        break;
    case GSQL_AGG_AVG: v.d += o.d; v.l += o.l; break;
    default: v.l = (long long)((unsigned long long)v.l + (unsigned long long)o.l); break;  // COUNT, COUNT_STAR, SUM0
    }
    v.has |= o.has;
}

__device__ __forceinline__ void derive_store(const AggDev &a, int gid, const DeriveVal &v) {
    switch (a.kind) {
    case GSQL_AGG_COUNT_STAR: case GSQL_AGG_COUNT: case GSQL_AGG_SUM0:
        if (v.l) atomicAdd(reinterpret_cast<unsigned long long *>(&a.l[gid]), (unsigned long long)v.l);
        return;
    default: break;
    }
    if (!v.has) return;
    switch (a.kind) {
    case GSQL_AGG_SUM:
        if (a.in_type == GSQL_T_FP64) atomicAdd(&a.d[gid], v.d);
        else {
            const unsigned long long old = atomicAdd(reinterpret_cast<unsigned long long *>(&a.l[gid]), (unsigned long long)v.l);
            const unsigned long long carry = old + (unsigned long long)v.l < old ? 1ULL : 0ULL;
            const unsigned long long hi = (unsigned long long)v.hi + carry;
            if (hi) atomicAdd(reinterpret_cast<unsigned long long *>(&a.hi[gid]), hi);
        }
        break;
    case GSQL_AGG_AVG:
        atomicAdd(&a.d[gid], v.d);
        atomicAdd(reinterpret_cast<unsigned long long *>(&a.l[gid]), (unsigned long long)v.l);
        break;
    case GSQL_AGG_MIN: atomicMin(reinterpret_cast<long long *>(&a.l[gid]), v.l); break;
    default: atomicMax(reinterpret_cast<long long *>(&a.l[gid]), v.l); break;
    }
    if (!ld_keep_u8(&a.has[gid], l2_policy_evict_last())) a.has[gid] = 1;  // the slot hint stays 0: always safe
}

// One parent group per lane; the warp is brought back together around the probe as in agg_rows.  Lanes whose parent
// groups fall into one child group fold their states into the lowest of them first (__match_any_sync on the child gid),
// so a child of one group (the grand total) takes one atomic per warp and state, not one per parent group.
template <int NK>
__global__ void __launch_bounds__(256) k_agg_derive(const __grid_constant__ AggParams P, const __grid_constant__ DeriveSrc S) {
    const int lane = threadIdx.x & 31;
    const int64_t stride = (int64_t)gridDim.x * blockDim.x;
    for (int64_t base = blockIdx.x * (int64_t)blockDim.x + (threadIdx.x - lane); base < S.ngroups; base += stride) {
        const int64_t g = base + lane;
        const bool live = g < S.ngroups;
        int gid = -1;
        if (live) {
            int64_t kv[GSQL_MAX_KEYS];
            bool kn[GSQL_MAX_KEYS];
            if constexpr (NK > 0) {
#pragma unroll
                for (int c = 0; c < NK; c++) {
                    kv[c] = S.gkey[c][g];
                    kn[c] = S.gnull[c][g] != 0;
                }
            } else {
#pragma unroll 1
                for (int c = 0; c < P.nkeys; c++) {
                    kv[c] = S.gkey[c][g];
                    kn[c] = S.gnull[c][g] != 0;
                }
            }
            gid = find_group_kv<NK>(P, kv, kn, digest_of_keys<NK>(P, kv, kn), true);
        }
        __syncwarp();
        const unsigned peers = __match_any_sync(0xffffffffu, gid);
        const int leader = __ffs(peers) - 1;
        const unsigned folded = __ballot_sync(0xffffffffu, live && lane != leader);  // warp-uniform
        for (int a = 0; a < P.naggs; a++) {
            const AggDev &ca = P.agg[a];
            DeriveVal v = derive_load(S.agg[a], g, live);
            for (unsigned m = folded; m; m &= m - 1) {
                const int j = __ffs(m) - 1;
                DeriveVal o;
                o.l = __shfl_sync(0xffffffffu, v.l, j);
                o.hi = __shfl_sync(0xffffffffu, v.hi, j);
                o.d = __shfl_sync(0xffffffffu, v.d, j);
                o.has = __shfl_sync(0xffffffffu, (int)v.has, j) != 0;
                if (lane == leader && ((peers >> j) & 1u)) derive_fold(ca, v, o);
            }
            if (live && lane == leader) derive_store(ca, gid, v);
        }
        __syncwarp();
    }
}

// The NULL or constant of a group column the set does not reference, over rows [0, n) of a device column.
__global__ void __launch_bounds__(256) k_gsagg_fill(void *data, uint8_t *nulls, int32_t type, int64_t value, int32_t is_null, int64_t n) {
    for (int64_t i = blockIdx.x * (int64_t)blockDim.x + threadIdx.x; i < n; i += (int64_t)gridDim.x * blockDim.x) {
        nulls[i] = is_null ? 1 : 0;
        if (type == GSQL_T_INT32) reinterpret_cast<int32_t *>(data)[i] = is_null ? 0 : (int32_t)value;
        else reinterpret_cast<int64_t *>(data)[i] = is_null ? 0 : value;
    }
}

struct GsSet {
    int32_t nref = 0;
    int32_t refk[GSQL_MAX_KEYS];  // the group columns (indices into the agg spec's groups) this set references, in order
    bool root = false;
    gsql_agg *agg = nullptr;      // keyed by the referenced input columns
};

struct gsql_gsagg {
    gsql_ctx *ctx;
    gsql_expand_spec ex;
    gsql_agg_spec spec;  // over the Expand output
    int32_t nout = 0;
    int32_t out_types[GSQL_MAX_COLS];
    GsSet set[GSQL_MAX_SETS];
    int32_t order[GSQL_MAX_SETS];  // finest first: every set a set derives from comes before it
    int64_t rows = 0;
    bool finished = false;
    bool failed = false;  // a finish that failed part-way: the handle is left unusable, never half-built
    int32_t cur_set = 0;
    ~gsql_gsagg() {
        for (auto &s : set) gsql_agg_destroy(s.agg);
    }
};

// Set t derives from set s: every group column t references has the same reference in s; between equal sets the later
// derives from the earlier.  *pk (may be null) receives, per key of t, the index of the same key among s's.
static bool gs_derives(const gsql_gsagg *G, int t, int s, int32_t *pk) {
    if (s == t) return false;
    const GsSet &T = G->set[t], &S = G->set[s];
    if (T.nref > S.nref || (T.nref == S.nref && s > t)) return false;
    for (int j = 0; j < T.nref; j++) {
        const int k = T.refk[j];
        const int gc = G->spec.groups[k];
        int at = -1;
        for (int q = 0; q < S.nref; q++)
            if (S.refk[q] == k && G->ex.proj[s][gc].col == G->ex.proj[t][gc].col) at = q;
        if (at < 0) return false;
        if (pk) pk[j] = at;
    }
    return true;
}

// The gsql_agg spec of set s over the Expand's input: its referenced columns as keys, the calls remapped.
static gsql_agg_spec gs_set_spec(const gsql_gsagg *G, int s, int64_t expected_groups) {
    gsql_agg_spec a;
    memset(&a, 0, sizeof(a));
    a.n_input_cols = G->ex.n_input_cols;
    for (int i = 0; i < G->ex.n_input_cols; i++) a.input_types[i] = G->ex.input_types[i];
    a.ngroups = G->set[s].nref;
    for (int j = 0; j < a.ngroups; j++) a.groups[j] = G->ex.proj[s][G->spec.groups[G->set[s].refk[j]]].col;
    a.naggs = G->spec.naggs;
    for (int i = 0; i < a.naggs; i++) {
        gsql_agg_call c = G->spec.aggs[i];
        for (int q = 0; q < c.ncols; q++) c.cols[q] = G->ex.proj[0][c.cols[q]].col;
        if (c.filter_arg >= 0) c.filter_arg = G->ex.proj[0][c.filter_arg].col;
        a.aggs[i] = c;
    }
    a.expected_groups = expected_groups;
    a.row_filter_col = -1;
    a.row_filter_op = GSQL_CMP_NONE;
    return a;
}

static gsql_status gs_check(gsql_ctx *ctx, const gsql_expand_spec &e, const gsql_agg_spec &s) {
    if (e.n_input_cols < 0 || e.n_input_cols > GSQL_MAX_COLS) return gsql_set_error(ctx, GSQL_E_INVALID, "bad expand input column count");
    for (int i = 0; i < e.n_input_cols; i++)
        if (e.input_types[i] < GSQL_T_INT32 || e.input_types[i] > GSQL_T_FP64) return gsql_set_error(ctx, GSQL_E_UNSUPPORTED, "expand input col %d type", i);
    if (e.nsets < 1 || e.nsets > GSQL_MAX_SETS) return gsql_set_error(ctx, GSQL_E_UNSUPPORTED, "%d grouping sets (1..%d)", e.nsets, GSQL_MAX_SETS);
    if (e.n_output_cols != s.n_input_cols) return gsql_set_error(ctx, GSQL_E_INVALID, "expand has %d output columns, the agg spec %d", e.n_output_cols, s.n_input_cols);
    for (int p = 0; p < e.nsets; p++)
        for (int c = 0; c < e.n_output_cols; c++) {
            const gsql_expand_item &it = e.proj[p][c];
            if (it.src == GSQL_EXPAND_INPUT) {
                if (it.col < 0 || it.col >= e.n_input_cols) return gsql_set_error(ctx, GSQL_E_INVALID, "projection %d col %d: input column out of range", p, c);
                if (e.input_types[it.col] != s.input_types[c])
                    return gsql_set_error(ctx, GSQL_E_UNSUPPORTED, "projection %d col %d: input type %d, output type %d", p, c, e.input_types[it.col], s.input_types[c]);
            } else if (it.src == GSQL_EXPAND_CONST) {
                if (s.input_types[c] == GSQL_T_FP64) return gsql_set_error(ctx, GSQL_E_UNSUPPORTED, "projection %d col %d: constant in a DOUBLE column", p, c);
                if (s.input_types[c] == GSQL_T_INT32 && (it.value < INT32_MIN || it.value > INT32_MAX))
                    return gsql_set_error(ctx, GSQL_E_INVALID, "projection %d col %d: INT constant out of range", p, c);
            } else if (it.src != GSQL_EXPAND_NULL) {
                return gsql_set_error(ctx, GSQL_E_INVALID, "projection %d col %d: source %d", p, c, it.src);
            }
        }
    if (s.n_derived != 0) return gsql_set_error(ctx, GSQL_E_UNSUPPORTED, "derived columns over an expand");
    if (s.row_filter_op != GSQL_CMP_NONE) return gsql_set_error(ctx, GSQL_E_UNSUPPORTED, "row filter over an expand");
    for (int i = 0; i < s.naggs; i++) {
        const gsql_agg_call &c = s.aggs[i];
        if (c.kind == GSQL_AGG_FIRST_VALUE || c.kind == GSQL_AGG_AVG_MERGE)
            return gsql_set_error(ctx, GSQL_E_UNSUPPORTED, "agg %d: kind %d over an expand", i, c.kind);
        int used[5], nused = 0;
        for (int q = 0; q < c.ncols && q < 4; q++) used[nused++] = c.cols[q];
        if (c.filter_arg >= 0) used[nused++] = c.filter_arg;
        for (int u = 0; u < nused; u++) {
            const int col = used[u];
            if (col < 0 || col >= e.n_output_cols) continue;  // agg_check_spec reports it
            for (int p = 0; p < e.nsets; p++)
                if (e.proj[p][col].src != GSQL_EXPAND_INPUT || e.proj[p][col].col != e.proj[0][col].col)
                    return gsql_set_error(ctx, GSQL_E_UNSUPPORTED, "agg %d: column %d is not the same input column in every set", i, col);
        }
    }
    bool keyed = false;  // a group column of pairwise distinct constants ($e) keeps the sets' groups apart
    for (int k = 0; k < s.ngroups && !keyed; k++) {
        const int gc = s.groups[k];
        if (gc < 0 || gc >= e.n_output_cols) break;  // agg_check_spec reports it
        bool ok = true;
        for (int p = 0; p < e.nsets && ok; p++) {
            ok = e.proj[p][gc].src == GSQL_EXPAND_CONST;
            for (int q = 0; q < p && ok; q++) ok = e.proj[q][gc].value != e.proj[p][gc].value;
        }
        keyed = ok;
    }
    if (!keyed) return gsql_set_error(ctx, GSQL_E_UNSUPPORTED, "no group column with a distinct constant in every set");
    return GSQL_OK;
}

extern "C" gsql_status gsql_gsagg_create(gsql_ctx *ctx, const gsql_expand_spec *expand, const gsql_agg_spec *spec, gsql_gsagg **out) {
    if (!ctx || !expand || !spec || !out) return GSQL_E_INVALID;
    if (ctx->sticky) return GSQL_E_CUDA;
    *out = nullptr;
    int32_t in_type[GSQL_MAX_AGGS], out_types[GSQL_MAX_COLS], nout = 0;
    GSQL_TRY(agg_check_spec(ctx, *spec, in_type, out_types, &nout));
    GSQL_TRY(gs_check(ctx, *expand, *spec));
    gsql_gsagg *G = new gsql_gsagg();
    G->ctx = ctx;
    gsql_ctx_retain(ctx);
    G->ex = *expand;
    G->spec = *spec;
    G->nout = nout;
    memcpy(G->out_types, out_types, sizeof(out_types));
    const int ns = expand->nsets;
    for (int s = 0; s < ns; s++) {
        GsSet &S = G->set[s];
        for (int k = 0; k < spec->ngroups; k++)
            if (expand->proj[s][spec->groups[k]].src == GSQL_EXPAND_INPUT) S.refk[S.nref++] = k;
    }
    for (int s = 0; s < ns; s++) G->order[s] = s;
    std::stable_sort(G->order, G->order + ns, [&](int a, int b) { return G->set[a].nref > G->set[b].nref; });
    gsql_status st = GSQL_OK;
    for (int t = 0; t < ns && st == GSQL_OK; t++) {
        bool root = true;
        for (int s = 0; s < ns && root; s++) root = !gs_derives(G, t, s, nullptr);
        G->set[t].root = root;
        if (root) {
            const gsql_agg_spec a = gs_set_spec(G, t, spec->expected_groups);
            st = gsql_agg_create(ctx, &a, &G->set[t].agg);
        }
    }
    if (st != GSQL_OK) {
        delete G;
        gsql_ctx_release(ctx);
        return st;
    }
    *out = G;
    return GSQL_OK;
}

extern "C" void gsql_gsagg_destroy(gsql_gsagg *G) {
    if (!G) return;
    gsql_ctx *ctx = G->ctx;
    delete G;  // each set's gsql_agg_destroy waits for its stream-ordered frees
    gsql_ctx_release(ctx);
}

extern "C" gsql_status gsql_gsagg_consume(gsql_gsagg *G, const gsql_batch *batch) {
    if (!G) return GSQL_E_INVALID;
    gsql_ctx *ctx = G->ctx;
    if (ctx->sticky) return GSQL_E_CUDA;
    if (G->finished || G->failed) return gsql_set_error(ctx, GSQL_E_STATE, "consume after finish");
    GSQL_TRY(validate_batch(ctx, batch, G->ex.n_input_cols, G->ex.input_types));
    if (batch->rows == 0) return GSQL_OK;
    GSQL_CUDA(ctx, cudaSetDevice(ctx->device));
    gsql_batch stripped;
    gsql_col stripped_cols[GSQL_MAX_COLS];
    GSQL_TRY(strip_zero_masks(ctx, batch, &stripped, stripped_cols));  // once, not once per root
    StagedBatch sb;  // a host batch is uploaded once and every root reads the same device copy
    GSQL_TRY(stage_batch(ctx, &stripped, &sb));
    gsql_col dcols[GSQL_MAX_COLS];
    for (int i = 0; i < sb.ncols; i++) {
        dcols[i].type = sb.cols[i].type;
        dcols[i].reserved = 0;
        dcols[i].data = const_cast<void *>(sb.cols[i].data);
        dcols[i].nulls = const_cast<uint8_t *>(sb.cols[i].nulls);
    }
    gsql_batch dev{batch->rows, sb.ncols, GSQL_MEM_DEVICE, dcols};
    for (int s = 0; s < G->ex.nsets; s++)
        if (G->set[s].root) GSQL_TRY(gsql_agg_consume(G->set[s].agg, &dev));
    G->rows += batch->rows;
    if (batch->mem == GSQL_MEM_HOST) GSQL_CUDA(ctx, cudaStreamSynchronize(ctx->stream));
    return GSQL_OK;
}

// Builds derived set t from its finished parent p (pk: t's keys among p's).
static gsql_status gs_derive(gsql_gsagg *G, int t, int p, const int32_t *pk) {
    gsql_ctx *ctx = G->ctx;
    gsql_agg *par = G->set[p].agg;
    const gsql_agg_spec a = gs_set_spec(G, t, par->ngroups > 1 ? par->ngroups : 1);  // the child never outgrows its parent
    GSQL_TRY(gsql_agg_create(ctx, &a, &G->set[t].agg));
    gsql_agg *ch = G->set[t].agg;
    if (par->ngroups == 0) {  // a parent without groups gives a child without groups (a grand total included)
        ch->ngroups = 0;
        return GSQL_OK;
    }
    AggParams P;
    agg_fill_params(ch, nullptr, &P);
    AggParams PP;
    agg_fill_params(par, nullptr, &PP);
    DeriveSrc S;
    memset(&S, 0, sizeof(S));
    S.ngroups = par->ngroups;
    for (int j = 0; j < ch->nkeys; j++) {
        S.gkey[j] = PP.gkey[pk[j]];
        S.gnull[j] = PP.gnull[pk[j]];
    }
    for (int i = 0; i < par->naggs; i++) S.agg[i] = PP.agg[i];
    {
        KernelScope ks(ctx, "agg_derive");
        const int grid = grid_rows(ctx, S.ngroups, 256, 8);
        switch (ch->nkeys) {  // the key count as a template argument keeps the key image in registers (see digest_of_keys)
        case 1: k_agg_derive<1><<<grid, 256, 0, ctx->stream>>>(P, S); break;
        case 2: k_agg_derive<2><<<grid, 256, 0, ctx->stream>>>(P, S); break;
        case 3: k_agg_derive<3><<<grid, 256, 0, ctx->stream>>>(P, S); break;
        default: k_agg_derive<0><<<grid, 256, 0, ctx->stream>>>(P, S); break;
        }
    }
    GSQL_CUDA(ctx, cudaGetLastError());
    unsigned long long h[C_COUNT];
    GSQL_TRY(agg_read_counters(ch, h));
    ch->ngroups = (int64_t)h[C_NGROUPS];
    if (h[C_FATAL]) {
        ctx->sticky = true;
        return gsql_set_error(ctx, GSQL_E_CAPACITY, "derived set %d: group arrays overflowed", t);
    }
    return GSQL_OK;
}

extern "C" gsql_status gsql_gsagg_finish(gsql_gsagg *G, int64_t *ngroups) {
    if (!G) return GSQL_E_INVALID;
    gsql_ctx *ctx = G->ctx;
    if (ctx->sticky) return GSQL_E_CUDA;
    GSQL_CUDA(ctx, cudaSetDevice(ctx->device));
    if (G->failed) return gsql_set_error(ctx, GSQL_E_STATE, "an earlier finish failed");
    if (!G->finished) {
        G->failed = true;  // until every set is built
        const int ns = G->ex.nsets;
        for (int s = 0; s < ns; s++)  // no row consumed: no set has a group (a root without keys starts with one)
            if (G->set[s].root && G->rows == 0) G->set[s].agg->ngroups = 0;
        for (int o = 0; o < ns; o++) {
            const int t = G->order[o];
            if (G->set[t].root) continue;
            int best = -1;
            int32_t best_pk[GSQL_MAX_KEYS], pk[GSQL_MAX_KEYS];
            for (int q = 0; q < o; q++) {  // the finished superset with the fewest groups
                const int s = G->order[q];
                if (gs_derives(G, t, s, pk) && (best < 0 || G->set[s].agg->ngroups < G->set[best].agg->ngroups)) {
                    best = s;
                    memcpy(best_pk, pk, sizeof(pk));
                }
            }
            if (best < 0) return gsql_set_error(ctx, GSQL_E_STATE, "set %d has no finished parent", t);
            GSQL_TRY(gs_derive(G, t, best, best_pk));
        }
        for (int s = 0; s < ns; s++) GSQL_TRY(gsql_agg_finish(G->set[s].agg, nullptr));
        for (int s = 0; s < ns; s++) {  // only the finished rows are read from here on: tables and states go back now
            gsql_agg *a = G->set[s].agg;
            a->slots.release();
            a->overflow.release();
            for (int k = 0; k < a->nkeys; k++) {
                a->gkey[k].release();
                a->gnull[k].release();
            }
            for (int i = 0; i < a->naggs; i++) {
                a->sl[i].release();
                a->shi[i].release();
                a->sd[i].release();
                a->shas[i].release();
            }
        }
        G->failed = false;
        G->finished = true;
        G->cur_set = 0;
    }
    if (ngroups) {
        int64_t n = 0;
        for (int s = 0; s < G->ex.nsets; s++) n += G->set[s].agg->ngroups;
        *ngroups = n;
    }
    return GSQL_OK;
}

extern "C" gsql_status gsql_gsagg_output_schema(gsql_gsagg *G, int32_t *ncols, int32_t *types) {
    if (!G || !ncols) return GSQL_E_INVALID;
    *ncols = G->nout;
    if (types)
        for (int i = 0; i < G->nout; i++) types[i] = G->out_types[i];
    return GSQL_OK;
}

extern "C" gsql_status gsql_gsagg_next(gsql_gsagg *G, gsql_batch *out, int64_t max_rows, int64_t *out_rows) {
    if (!G || !out || !out_rows) return GSQL_E_INVALID;
    gsql_ctx *ctx = G->ctx;
    if (ctx->sticky) return GSQL_E_CUDA;
    if (!G->finished) return gsql_set_error(ctx, GSQL_E_STATE, "next before finish");
    GSQL_TRY(validate_batch(ctx, out, G->nout, G->out_types));
    for (int c = 0; c < G->nout; c++)
        if (!out->cols[c].nulls) return gsql_set_error(ctx, GSQL_E_INVALID, "grouping sets output column %d needs a nulls buffer", c);
    GSQL_CUDA(ctx, cudaSetDevice(ctx->device));
    const cudaMemcpyKind kind = out->mem == GSQL_MEM_DEVICE ? cudaMemcpyDeviceToDevice : cudaMemcpyDeviceToHost;
    const int nk = G->spec.ngroups;
    int64_t done = 0;
    while (done < max_rows && G->cur_set < G->ex.nsets) {
        const int s = G->cur_set;
        gsql_agg *a = G->set[s].agg;
        int64_t n = a->ngroups - a->cursor;
        if (n <= 0) {
            G->cur_set++;
            continue;
        }
        if (n > max_rows - done) n = max_rows - done;
        int j = 0;  // the set's next referenced key
        for (int c = 0; c < G->nout; c++) {
            const int w = gsql_type_width(G->out_types[c]);
            char *dst = (char *)out->cols[c].data + (size_t)done * w;
            uint8_t *dnull = out->cols[c].nulls + done;
            int src = -1;  // column of the set's own result
            if (c >= nk) src = G->set[s].nref + (c - nk);
            else if (j < G->set[s].nref && G->set[s].refk[j] == c) src = j++;
            if (src >= 0) {
                GSQL_CUDA(ctx, cudaMemcpyAsync(dst, (char *)a->out_data[src].p + (size_t)a->cursor * w, (size_t)n * w, kind, ctx->stream));
                GSQL_CUDA(ctx, cudaMemcpyAsync(dnull, (char *)a->out_nulls[src].p + a->cursor, (size_t)n, kind, ctx->stream));
                continue;
            }
            const gsql_expand_item &it = G->ex.proj[s][G->spec.groups[c]];
            const bool is_null = it.src == GSQL_EXPAND_NULL;
            if (out->mem == GSQL_MEM_DEVICE) {
                KernelScope ks(ctx, "gsagg_fill");
                k_gsagg_fill<<<grid_rows(ctx, n, 256, 4), 256, 0, ctx->stream>>>(dst, dnull, G->out_types[c], it.value, is_null, n);
                GSQL_CUDA(ctx, cudaGetLastError());
            } else {
                memset(dnull, is_null ? 1 : 0, (size_t)n);
                for (int64_t r = 0; r < n; r++) {
                    if (G->out_types[c] == GSQL_T_INT32) reinterpret_cast<int32_t *>(dst)[r] = is_null ? 0 : (int32_t)it.value;
                    else reinterpret_cast<int64_t *>(dst)[r] = is_null ? 0 : it.value;
                }
            }
        }
        a->cursor += n;
        done += n;
    }
    *out_rows = done;
    out->rows = done;
    if (out->mem == GSQL_MEM_HOST) GSQL_CUDA(ctx, cudaStreamSynchronize(ctx->stream));
    return GSQL_OK;
}
