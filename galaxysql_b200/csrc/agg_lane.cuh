// agg_lane.cuh — LANE-private accumulators for very low cardinality group-by (the TPC-H Q1 shape: 4-6 groups, 8
// aggregates), included by agg.cu after agg_fast.cuh.
//
// k_agg_smem (agg_fast.cuh) keeps one accumulator per (warp, group) and pays for it with warp-wide peer reductions:
// dozens of warp-instructions per ROW on the Q1 shape, i.e. it is issue-bound.
// Here every LANE owns a private copy of every accumulator of every group of its warp:
//
//     acc[(slot * nacc + a) * 32 + lane]        (8 bytes each, shared memory)
//
// A row is then processed by its lane alone: find the slot of its key in the warp's small key dictionary (broadcast
// reads), and for each accumulator one LDS / DADD / STS on the lane's own cell — no atomics, no shuffles, no bank
// conflicts (lanes hit 32 different banks whatever the slot).  Accumulators are de-duplicated on the host: SUM(x) and
// AVG(x) share one fp64 sum, and every "count of non-NULL x" collapses into the group's row counter when the batch
// carries no NULL buffer for x (Q1: 8 aggregates -> 5 sums + 1 counter).  Every plan entry (key component, accumulator)
// is decoded once per step and applied to the R rows a lane owns in that step; the loads of the warp's next step are
// issued before the current step is accumulated.  16 warps per SM x R = 2 measured faster on the Q1 shape than
// 8 warps x R = 4 (the kernel is issue-latency bound — 2 warps per scheduler cannot cover the dependent
// LDS / DADD / STS chains), so shared memory is split 16 ways: S = 6 groups per warp at Q1's 6 accumulators.
// When a warp finishes, each accumulator is reduced over the lanes with shuffles and merged into the global table
// (find_group_kv + L2 atomics) exactly like the shared-memory path.
//
// Adaptive like the other fast path: a row whose key does not fit the warp's S-slot dictionary takes the generic path on
// the spot and is counted in C_FALLBACK; the host drops back to k_agg_smem / the generic kernel when that is common.
//
// Reference behaviour: AggOpenHashMap.putChunk (EX/operator/util/AggOpenHashMap.java:100-139) and the aggregators
// (restated by the CPU checker under tests) — same groups, same NULL rules; floating sums are added in a different order (within the
// north_star's 1e-6 relative tolerance), integer results are bit-exact.
#pragma once

namespace {

constexpr int LA_THREADS = 512;
constexpr int LA_WARPS = LA_THREADS / 32;
constexpr int LA_R = 2;          // rows per lane per step
constexpr int LA_MAX_USED = 8;   // input columns touched
constexpr int LA_MAX_ACC = 12;   // lane-private accumulators per group
constexpr int LA_MAX_S = 16;     // dictionary slots per warp
enum { LA_FSUM = 0, LA_CNT = 1, LA_CNT_STAR = 2, LA_ISUM0 = 3, LA_MIN = 4, LA_MAX = 5 };

// A value the kernel reads per row: a staged input column or a fused derived expression over staged columns
// (VectorizedProjectExec replacement, gsql_derived_col).  u* are staging rows, f* say "the column is DOUBLE".
struct LaneRef {
    int8_t kind;  // 0 plain, GSQL_EXPR_MUL_1MINUS, GSQL_EXPR_MUL_1MINUS_1PLUS
    int8_t ua, ub, uc;
    int8_t fa, fb, fc;
    int8_t pad;
};

struct LanePlan {
    int32_t S, nacc;
    int32_t nused;
    int32_t used[LA_MAX_USED];
    int8_t colmap[GSQL_MAX_COLS];  // input column -> staging row, -1 = unused
    int32_t any_nulls;             // some used column carries a NULL buffer in this batch
    // accumulators: kind, argument, and the staging rows whose NULL flag vetoes the row for this accumulator (bit mask)
    int8_t acc_kind[LA_MAX_ACC];
    int8_t acc_fp[LA_MAX_ACC];       // MIN / MAX: argument is fp64 (sortable image)
    int8_t acc_ncols[LA_MAX_ACC];
    int16_t acc_cols[LA_MAX_ACC][4];  // argument column(s) as the spec names them (de-duplication key; host only)
    LaneRef acc_ref[LA_MAX_ACC];
    uint32_t acc_nullmask[LA_MAX_ACC];
    // per aggregate: the accumulator holding its value and the one counting its contributing rows
    int8_t agg_val[GSQL_MAX_AGGS];
    int8_t agg_cnt[GSQL_MAX_AGGS];
    // 16-byte key image: per key column its byte offset, width and the offset of its NULL byte (-1: not nullable)
    int8_t key_off[GSQL_MAX_KEYS], key_w[GSQL_MAX_KEYS], key_noff[GSQL_MAX_KEYS];
    int8_t key_u[GSQL_MAX_KEYS], key_fp[GSQL_MAX_KEYS];
    int8_t rf_u;  // staging row of the row-filter column
    int8_t key_bytes;  // bytes of the key image in use (<= 16)
    // shared memory of one warp
    int32_t off_dict, off_n, off_acc, off_red, off_stage, warp_bytes, total;
};

__device__ __forceinline__ double warp_sum_f64(double v) {
#pragma unroll
    for (int d = 16; d > 0; d >>= 1) v += __shfl_xor_sync(0xffffffffu, v, d);
    return v;
}
__device__ __forceinline__ long long warp_sum_i64(long long v) {
#pragma unroll
    for (int d = 16; d > 0; d >>= 1) v = (long long)((unsigned long long)v + (unsigned long long)__shfl_xor_sync(0xffffffffu, v, d));
    return v;
}
__device__ __forceinline__ long long warp_minmax_i64(long long v, bool mx) {
#pragma unroll
    for (int d = 16; d > 0; d >>= 1) {
        long long o = __shfl_xor_sync(0xffffffffu, v, d);
        v = mx ? (o > v ? o : v) : (o < v ? o : v);
    }
    return v;
}

__global__ void __launch_bounds__(LA_THREADS, 1) k_agg_lane(const __grid_constant__ AggParams P, const __grid_constant__ LanePlan L) {
    extern __shared__ __align__(16) char sm_all[];
    const int lane = threadIdx.x & 31;
    char *sm = sm_all + (size_t)(threadIdx.x >> 5) * L.warp_bytes;
    unsigned long long *dict = reinterpret_cast<unsigned long long *>(sm + L.off_dict);  // [S][2]
    volatile int *ndict = reinterpret_cast<volatile int *>(sm + L.off_n);
    long long *acc = reinterpret_cast<long long *>(sm + L.off_acc);
    unsigned long long *sval = reinterpret_cast<unsigned long long *>(sm + L.off_stage) + lane;  // [nused][R][32], this lane's cells

    // ---- init: identities of the lane's cells, empty dictionary (one preset group when there is no GROUP BY)
    for (int s = 0; s < L.S; s++)
        for (int a = 0; a < L.nacc; a++) {
            long long init = L.acc_kind[a] == LA_MIN ? 0x7fffffffffffffffLL : L.acc_kind[a] == LA_MAX ? (long long)0x8000000000000000ULL : 0;
            acc[(s * L.nacc + a) * 32 + lane] = init;
        }
    if (lane == 0) {
        *ndict = P.nkeys == 0 ? 1 : 0;
        dict[0] = 0;
        dict[1] = 0;
    }
    __syncwarp();

    const int64_t warps_total = (int64_t)gridDim.x * LA_WARPS;
    const int64_t warp_id = (int64_t)blockIdx.x * LA_WARPS + (threadIdx.x >> 5);
    // staged cell of staging row u, row k of this lane: sval[(u * LA_R + k) * 32]
    auto st_f64 = [&](int u, bool isfp, int k) -> double {
        unsigned long long v = sval[(u * LA_R + k) * 32];
        return isfp ? __longlong_as_double((long long)v) : (double)(long long)v;
    };
    auto ref_f64 = [&](const LaneRef &r, int k) -> double {
        double x = st_f64(r.ua, r.fa != 0, k);
        if (r.kind != 0) {
            x = x * (1.0 - st_f64(r.ub, r.fb != 0, k));
            if (r.kind == GSQL_EXPR_MUL_1MINUS_1PLUS) x = x * (1.0 + st_f64(r.uc, r.fc != 0, k));
        }
        return x;
    };

    unsigned int fallback_rows = 0;
    // Software pipeline: the loads of the warp's NEXT step are issued right after the current step's values have been
    // moved from registers to the staging cells, so their HBM latency overlaps the accumulate phase (the first profile
    // of this kernel had ~45 % of its stall samples on the first use of the loaded values).
    unsigned long long raw[LA_MAX_USED][LA_R];
    uint8_t nul[LA_MAX_USED][LA_R];
    auto issue_loads = [&](int64_t b) {
        const bool full = b + 32 * LA_R <= P.rows;  // warp-uniform: no per-row bounds checks on full steps
#pragma unroll
        for (int u = 0; u < LA_MAX_USED; u++) {
            if (u < L.nused) {
                const DCol &col = P.in.c[L.used[u]];
                const bool is32 = col.type == GSQL_T_INT32;
                const char *dp = reinterpret_cast<const char *>(col.data) + (P.row0 + b + lane) * (is32 ? 4 : 8);
                const uint8_t *np = col.nulls ? col.nulls + P.row0 + b + lane : nullptr;
#pragma unroll
                for (int k = 0; k < LA_R; k++) {
                    raw[u][k] = 0;
                    nul[u][k] = 0;
                    if (full || b + k * 32 + lane < P.rows) {
                        if (is32) raw[u][k] = (unsigned long long)(unsigned int)ld_stream_4(dp + k * 32 * 4);  // sign-extended when staged
                        else raw[u][k] = (unsigned long long)ld_stream_8(dp + k * 32 * 8);
                        if (np) nul[u][k] = np[k * 32];
                    }
                }
            }
        }
    };
    const int64_t b0 = warp_id * (32 * LA_R), bstride = warps_total * (32 * LA_R);
    if (b0 < P.rows) issue_loads(b0);
    for (int64_t b = b0; b < P.rows; b += bstride) {
        // ---- 1. values staged in the lane's own cells, NULL flags kept as one bit per staging row in a register
        unsigned int nullbits[LA_R];
#pragma unroll
        for (int k = 0; k < LA_R; k++) nullbits[k] = 0;
#pragma unroll
        for (int u = 0; u < LA_MAX_USED; u++) {
            if (u < L.nused) {
                const bool is32 = P.in.c[L.used[u]].type == GSQL_T_INT32;
#pragma unroll
                for (int k = 0; k < LA_R; k++) {
                    sval[(u * LA_R + k) * 32] = is32 ? (unsigned long long)(long long)(int)(unsigned int)raw[u][k] : raw[u][k];
                    if (L.any_nulls) nullbits[k] |= (nul[u][k] ? 1u : 0u) << u;
                }
            }
        }
        if (b + bstride < P.rows) issue_loads(b + bstride);
        // ---- 2. the R rows side by side (each lane its own rows); every plan entry is decoded once per step
        bool live[LA_R];
#pragma unroll
        for (int k = 0; k < LA_R; k++) live[k] = b + k * 32 + lane < P.rows;
        if (P.rf_op != GSQL_CMP_NONE) {
            const int u = L.rf_u;
#pragma unroll
            for (int k = 0; k < LA_R; k++) {
                const long long v = (long long)sval[(u * LA_R + k) * 32];  // INT / BIGINT only (checked at create)
                bool pass;
                switch (P.rf_op) {
                case GSQL_CMP_LE: pass = v <= P.rf_value; break;
                case GSQL_CMP_LT: pass = v < P.rf_value; break;
                case GSQL_CMP_GE: pass = v >= P.rf_value; break;
                case GSQL_CMP_GT: pass = v > P.rf_value; break;
                case GSQL_CMP_EQ: pass = v == P.rf_value; break;
                default: pass = v != P.rf_value; break;
                }
                live[k] = live[k] && pass && !((nullbits[k] >> u) & 1u);
            }
        }
        // 16-byte key image: canonical values (NULL -> 0, NaN / -0.0 canonical) and NULL bytes
        unsigned long long lo[LA_R], hi[LA_R];
#pragma unroll
        for (int k = 0; k < LA_R; k++) lo[k] = hi[k] = 0;
#pragma unroll 1
        for (int c = 0; c < P.nkeys; c++) {
            const int u = L.key_u[c], off = L.key_off[c], noff = L.key_noff[c];
            const bool isfp = L.key_fp[c] != 0, w4 = L.key_w[c] == 4;
#pragma unroll
            for (int k = 0; k < LA_R; k++) {
                long long v = (long long)sval[(u * LA_R + k) * 32];
                const bool kn = (nullbits[k] >> u) & 1u;
                if (isfp) {
                    double x = __longlong_as_double(v);
                    if (x != x) v = 0x7ff8000000000000LL;
                    else if (x == 0.0) v = 0;
                }
                if (kn) v = 0;
                const unsigned long long bits = w4 ? (unsigned long long)(unsigned int)v : (unsigned long long)v;
                if (off < 8) lo[k] |= bits << (off * 8);  // components never straddle the two words (host layout)
                else hi[k] |= bits << ((off - 8) * 8);
                if (noff >= 0 && kn) {
                    if (noff < 8) lo[k] |= 1ULL << (noff * 8);
                    else hi[k] |= 1ULL << ((noff - 8) * 8);
                }
            }
        }
        int slot[LA_R];
#pragma unroll
        for (int k = 0; k < LA_R; k++) slot[k] = live[k] ? -1 : -3;
        {
            const int n = *ndict;
            if (L.key_bytes <= 8) {  // the whole image is in the low word (hi == 0 everywhere)
#pragma unroll 1
                for (int s = 0; s < n; s++) {
                    const unsigned long long d0 = dict[2 * s];
#pragma unroll
                    for (int k = 0; k < LA_R; k++)
                        if (lo[k] == d0 && slot[k] == -1) slot[k] = s;
                }
            } else {
#pragma unroll 1
                for (int s = 0; s < n; s++) {
                    const unsigned long long d0 = dict[2 * s], d1 = dict[2 * s + 1];
#pragma unroll
                    for (int k = 0; k < LA_R; k++)
                        if (lo[k] == d0 && hi[k] == d1 && slot[k] == -1) slot[k] = s;
                }
            }
        }
#pragma unroll
        for (int k = 0; k < LA_R; k++) {
            unsigned need = __ballot_sync(0xffffffffu, slot[k] == -1);
            while (need) {  // a new key: the first lane that holds it appends it (or reports the dictionary full)
                const int leader = __ffs(need) - 1;
                const unsigned long long l0 = __shfl_sync(0xffffffffu, lo[k], leader), l1 = __shfl_sync(0xffffffffu, hi[k], leader);
                const int n = *ndict;
                int ns = -2;
                for (int s = 0; s < n; s++)  // appended by an earlier row of this step?
                    if (dict[2 * s] == l0 && dict[2 * s + 1] == l1) ns = s;
                const bool append = ns == -2 && n < L.S;
                if (append) ns = n;
                __syncwarp();  // every lane has read the dictionary before the leader extends it
                if (lane == leader && append) {
                    dict[2 * n] = l0;
                    dict[2 * n + 1] = l1;
                    *ndict = n + 1;
                }
                __syncwarp();
                if (slot[k] == -1 && lo[k] == l0 && hi[k] == l1) slot[k] = ns;
                need = __ballot_sync(0xffffffffu, slot[k] == -1);
            }
            if (slot[k] == -2) {  // does not fit this warp's dictionary: the generic path, right here
                fallback_rows++;
                int64_t kv[GSQL_MAX_KEYS];
                bool kn[GSQL_MAX_KEYS];
                for (int c = 0; c < P.nkeys; c++) {
                    const int off = L.key_off[c], noff = L.key_noff[c];
                    unsigned long long bits = (off < 8 ? lo[k] >> (off * 8) : hi[k] >> ((off - 8) * 8));
                    kv[c] = L.key_w[c] == 4 ? (int64_t)(int32_t)(unsigned int)bits : (int64_t)bits;
                    kn[c] = noff >= 0 && (((noff < 8 ? lo[k] >> (noff * 8) : hi[k] >> ((noff - 8) * 8)) & 0xff) != 0);
                }
                const int64_t r = P.row0 + b + k * 32 + lane;
                int gid = find_group_kv(P, kv, kn, digest_of_keys(P, kv, kn));
                if (gid < 0) {
                    unsigned long long o = atomicAdd(&P.counters[C_OVERFLOW], 1ULL);
                    P.overflow_rows[o] = r;
                } else {
                    for (int a = 0; a < P.naggs; a++) accumulate(P, P.agg[a], gid, r);
                }
            }
        }
        // accumulators: one decode per accumulator, then the R rows
        long long *cell[LA_R];
#pragma unroll
        for (int k = 0; k < LA_R; k++) cell[k] = acc + (size_t)(slot[k] > 0 ? slot[k] : 0) * L.nacc * 32 + lane;
#pragma unroll 1
        for (int a = 0; a < L.nacc; a++) {
            const int kind = L.acc_kind[a];
            const unsigned int nm = L.acc_nullmask[a];
            const LaneRef ref = L.acc_ref[a];
            switch (kind) {
            case LA_CNT_STAR:
            case LA_CNT:
#pragma unroll
                for (int k = 0; k < LA_R; k++)
                    if (slot[k] >= 0 && !(nullbits[k] & nm)) cell[k][a * 32] += 1;
                break;
            case LA_FSUM:
#pragma unroll
                for (int k = 0; k < LA_R; k++)
                    if (slot[k] >= 0 && !(nullbits[k] & nm)) {
                        double *c = reinterpret_cast<double *>(cell[k] + a * 32);
                        *c += ref_f64(ref, k);
                    }
                break;
            case LA_ISUM0:
#pragma unroll
                for (int k = 0; k < LA_R; k++)
                    if (slot[k] >= 0 && !(nullbits[k] & nm)) {
                        const long long v = ref.kind == 0 && !ref.fa ? (long long)sval[(ref.ua * LA_R + k) * 32] : (long long)ref_f64(ref, k);
                        cell[k][a * 32] = (long long)((unsigned long long)cell[k][a * 32] + (unsigned long long)v);
                    }
                break;
            default: {
                const bool mx = kind == LA_MAX;
#pragma unroll
                for (int k = 0; k < LA_R; k++)
                    if (slot[k] >= 0 && !(nullbits[k] & nm)) {
                        long long v;
                        if (L.acc_fp[a]) v = dbl_sortable(ref_f64(ref, k), mx);
                        else v = ref.kind == 0 && !ref.fa ? (long long)sval[(ref.ua * LA_R + k) * 32] : (long long)ref_f64(ref, k);
                        const long long c0 = cell[k][a * 32];
                        cell[k][a * 32] = mx ? (v > c0 ? v : c0) : (v < c0 ? v : c0);
                    }
            }
            }
        }
        __syncwarp();  // keep the warp converged before the staging cells are rewritten
    }
    if (fallback_rows) atomicAdd(&P.counters[C_FALLBACK], (unsigned long long)fallback_rows);
    __syncwarp();
    // ---- merge: reduce every accumulator over the lanes, then one lane folds the group into the global table
    long long *red = reinterpret_cast<long long *>(sm + L.off_red);  // [nacc]
    const int n = *ndict;
    for (int s = 0; s < n; s++) {
        for (int a = 0; a < L.nacc; a++) {
            long long v = acc[(s * L.nacc + a) * 32 + lane];
            const int kind = L.acc_kind[a];
            if (kind == LA_FSUM) v = __double_as_longlong(warp_sum_f64(__longlong_as_double(v)));
            else if (kind == LA_MIN || kind == LA_MAX) v = warp_minmax_i64(v, kind == LA_MAX);
            else v = warp_sum_i64(v);
            if (lane == 0) red[a] = v;
        }
        __syncwarp();
        if (lane == 0) {
            int64_t kv[GSQL_MAX_KEYS];
            bool kn[GSQL_MAX_KEYS];
            for (int c = 0; c < P.nkeys; c++) {
                const int off = L.key_off[c];
                unsigned long long bits = dict[2 * s + (off >> 3)] >> ((off & 7) * 8);
                kv[c] = L.key_w[c] == 4 ? (int64_t)(int32_t)(unsigned int)bits : (int64_t)bits;
                kn[c] = L.key_noff[c] >= 0 && ((dict[2 * s + (L.key_noff[c] >> 3)] >> ((L.key_noff[c] & 7) * 8)) & 0xff) != 0;
            }
            // a group whose rows contributed to no aggregate still has to exist; the merge may exceed gcap by at most
            // warps x S groups: covered by the arrays' slack (ignore_cap)
            const int gid = P.nkeys == 0 ? 0 : find_group_kv(P, kv, kn, digest_of_keys(P, kv, kn), true);
            for (int a = 0; a < P.naggs; a++) {
                const int kind = P.agg[a].kind;
                const long long cnt = L.agg_cnt[a] >= 0 ? red[L.agg_cnt[a]] : 0;
                SState st;
                st.x = L.agg_val[a] >= 0 ? red[L.agg_val[a]] : 0;  // a DOUBLE sum's bits
                st.l = kind == GSQL_AGG_SUM0 || kind == GSQL_AGG_MIN || kind == GSQL_AGG_MAX ? st.x : cnt;
                st.has = cnt != 0;
                state_merge(P.agg[a], gid, st);
            }
        }
        __syncwarp();
    }
}

}  // namespace

// Shape check at create time (independent of which columns carry NULL buffers).
static void agg_lane_check(AggFront *F, const gsql_agg_spec &spec, int nkeys, int naggs, const gsql_agg_call *aggs, const int32_t *in_type) {
    *F = AggFront{};
    int key_bytes = 0;
    for (int k = 0; k < nkeys; k++) key_bytes += spec.input_types[spec.groups[k]] == GSQL_T_INT32 ? 4 : 8;
    if (key_bytes > 16) return;
    for (int a = 0; a < naggs; a++) {
        if (aggs[a].filter_arg >= 0) return;                                     // per-aggregate FILTER stays on the other paths
        if (aggs[a].kind == GSQL_AGG_SUM && in_type[a] != GSQL_T_FP64) return;  // exact 128-bit SUM(int) stays generic
    }
    // the TPC-H Q1 shape is the target: a handful of groups.  expected_groups is the planner's hint (0 = unknown)
    if (spec.expected_groups > 4096) return;
    F->shape_ok = F->enabled = true;
}

// Per-batch plan: de-duplicated accumulators, key image, shared-memory layout.  false = this batch takes another path.
static bool agg_lane_plan(LanePlan *Lp, const gsql_agg_spec &spec, int nkeys, int naggs, const gsql_agg_call *aggs, const int32_t *in_type,
                          const DColSet &in) {
    LanePlan &L = *Lp;
    memset(&L, 0, sizeof(L));
    for (int c = 0; c < GSQL_MAX_COLS; c++) L.colmap[c] = -1;
    bool too_many = false;
    auto use1 = [&](int col) {
        if (L.colmap[col] >= 0) return;
        if (L.nused == LA_MAX_USED) { too_many = true; return; }
        L.colmap[col] = (int8_t)L.nused;
        L.used[L.nused++] = col;
        if (in.c[col].nulls) L.any_nulls = 1;
    };
    auto use = [&](int col) {
        if (col < 0) return;
        if (col >= spec.n_input_cols) {
            const gsql_derived_col &d = spec.derived[col - spec.n_input_cols];
            use1(d.a);
            use1(d.b);
            if (d.kind == GSQL_EXPR_MUL_1MINUS_1PLUS) use1(d.c);
        } else {
            use1(col);
        }
    };
    auto nullable = [&](int col) -> bool {
        if (col >= spec.n_input_cols) {
            const gsql_derived_col &d = spec.derived[col - spec.n_input_cols];
            return in.c[d.a].nulls || in.c[d.b].nulls || (d.kind == GSQL_EXPR_MUL_1MINUS_1PLUS && in.c[d.c].nulls);
        }
        return in.c[col].nulls != nullptr;
    };
    auto make_ref = [&](int col, LaneRef *r, uint32_t *nullmask) {  // after use(col)
        memset(r, 0, sizeof(*r));
        auto bit = [&](int c) { if (in.c[c].nulls) *nullmask |= 1u << L.colmap[c]; };
        if (col >= spec.n_input_cols) {
            const gsql_derived_col &d = spec.derived[col - spec.n_input_cols];
            r->kind = (int8_t)d.kind;
            r->ua = L.colmap[d.a]; r->fa = spec.input_types[d.a] == GSQL_T_FP64;
            r->ub = L.colmap[d.b]; r->fb = spec.input_types[d.b] == GSQL_T_FP64;
            bit(d.a);
            bit(d.b);
            if (d.kind == GSQL_EXPR_MUL_1MINUS_1PLUS) {
                r->uc = L.colmap[d.c]; r->fc = spec.input_types[d.c] == GSQL_T_FP64;
                bit(d.c);
            }
        } else {
            r->ua = L.colmap[col]; r->fa = spec.input_types[col] == GSQL_T_FP64;
            bit(col);
        }
    };
    // key image
    int off = 0;
    for (int k = 0; k < nkeys; k++) {  // 8-byte components first so that nothing straddles the two words
        if (spec.input_types[spec.groups[k]] == GSQL_T_INT32) continue;
        L.key_off[k] = (int8_t)off;
        L.key_w[k] = 8;
        off += 8;
    }
    for (int k = 0; k < nkeys; k++) {
        if (spec.input_types[spec.groups[k]] != GSQL_T_INT32) continue;
        L.key_off[k] = (int8_t)off;
        L.key_w[k] = 4;
        off += 4;
    }
    for (int k = 0; k < nkeys; k++) {
        L.key_noff[k] = -1;
        if (in.c[spec.groups[k]].nulls) L.key_noff[k] = (int8_t)off++;
        use(spec.groups[k]);
        if (too_many) return false;
        L.key_u[k] = L.colmap[spec.groups[k]];
        L.key_fp[k] = spec.input_types[spec.groups[k]] == GSQL_T_FP64;
    }
    if (off > 16) return false;
    L.key_bytes = (int8_t)off;
    if (spec.row_filter_op != GSQL_CMP_NONE) {
        use(spec.row_filter_col);
        if (too_many) return false;
        L.rf_u = L.colmap[spec.row_filter_col];
    }
    // accumulators
    auto find_acc = [&](int kind, int fp, int ncols, const int32_t *cols) -> int {
        for (int a = 0; a < L.nacc; a++) {
            if (L.acc_kind[a] != kind || L.acc_fp[a] != fp || L.acc_ncols[a] != ncols) continue;
            bool same = true;
            for (int q = 0; q < ncols; q++) same = same && L.acc_cols[a][q] == cols[q];
            if (same) return a;
        }
        if (L.nacc == LA_MAX_ACC) { too_many = true; return -1; }
        const int a = L.nacc++;
        L.acc_kind[a] = (int8_t)kind;
        L.acc_fp[a] = (int8_t)fp;
        L.acc_ncols[a] = (int8_t)ncols;
        for (int q = 0; q < ncols; q++) L.acc_cols[a][q] = (int16_t)cols[q];
        return a;
    };
    auto counter_of = [&](int ncols, const int32_t *cols) -> int {  // rows of the group whose arguments are all non-NULL
        bool any = false;
        for (int q = 0; q < ncols; q++) any = any || nullable(cols[q]);
        if (!any) return find_acc(LA_CNT_STAR, 0, 0, nullptr);
        return find_acc(LA_CNT, 0, ncols, cols);
    };
    for (int a = 0; a < naggs && !too_many; a++) {
        const gsql_agg_call &c = aggs[a];
        for (int q = 0; q < c.ncols; q++) use(c.cols[q]);
        L.agg_val[a] = -1;
        L.agg_cnt[a] = -1;
        switch (c.kind) {
        case GSQL_AGG_COUNT_STAR: L.agg_cnt[a] = (int8_t)find_acc(LA_CNT_STAR, 0, 0, nullptr); break;
        case GSQL_AGG_COUNT: L.agg_cnt[a] = (int8_t)counter_of(c.ncols, c.cols); break;
        case GSQL_AGG_SUM:
        case GSQL_AGG_AVG:
            L.agg_val[a] = (int8_t)find_acc(LA_FSUM, 0, 1, c.cols);
            L.agg_cnt[a] = (int8_t)counter_of(1, c.cols);
            break;
        case GSQL_AGG_SUM0: L.agg_val[a] = (int8_t)find_acc(LA_ISUM0, 0, 1, c.cols); break;
        case GSQL_AGG_MIN:
        case GSQL_AGG_MAX:
            L.agg_val[a] = (int8_t)find_acc(c.kind == GSQL_AGG_MIN ? LA_MIN : LA_MAX, in_type[a] == GSQL_T_FP64 ? 1 : 0, 1, c.cols);
            L.agg_cnt[a] = (int8_t)counter_of(1, c.cols);
            break;
        default: return false;
        }
    }
    if (too_many) return false;
    if (L.nacc == 0) find_acc(LA_CNT_STAR, 0, 0, nullptr);  // GROUP BY without aggregates: the groups must still appear
    for (int a = 0; a < L.nacc; a++) {
        L.acc_nullmask[a] = 0;
        memset(&L.acc_ref[a], 0, sizeof(LaneRef));
        for (int q = L.acc_ncols[a] - 1; q >= 0; q--) make_ref(L.acc_cols[a][q], &L.acc_ref[a], &L.acc_nullmask[a]);  // ref = first argument
    }
    // shared memory of one warp: <= ~26 KB so that 8 warps fit one SM
    const int stage = L.nused * LA_R * 32 * 8;
    const int budget = (208 * 1024) / LA_WARPS - stage - 16 - LA_MAX_S * 16 - LA_MAX_ACC * 8;
    int S = nkeys == 0 ? 1 : budget / (L.nacc * 256);
    if (S > LA_MAX_S) S = LA_MAX_S;
    if (S < (nkeys == 0 ? 1 : 4)) return false;
    L.S = S;
    int o = 0;
    L.off_acc = o;   o += S * L.nacc * 256;
    L.off_stage = o; o += stage;
    L.off_dict = o;  o += S * 16;
    L.off_red = o;   o += LA_MAX_ACC * 8;
    L.off_n = o;     o += 16;
    L.warp_bytes = (o + 15) & ~15;
    L.total = L.warp_bytes * LA_WARPS;
    return true;
}
