// agg_fast.cuh — shared-memory privatised group-by for low-cardinality keys (the TPC-H Q1 shape), included by agg.cu.
//
// Every WARP owns a small open-addressing table {key values, NULL flags, accumulators} in shared memory.  A warp
// step takes 32 rows: all the row's input columns are loaded with every load in flight and staged in a warp-private
// strip; each lane finds (or inserts) its key's slot in the warp table, lanes with the same slot are grouped with
// __match_any_sync, the group's values are reduced inside the warp with shuffles, and ONE lane per distinct key
// updates the accumulators with plain read-modify-writes — no atomics at all on the hot path (a CTA-shared table
// with shared-memory fp64 atomics was slower on the Q1 shape: CAS-loop contention on 6 hot slots).
// When a warp finishes its rows its <= S partial groups are merged into the global table (find_group_kv + L2 atomics).
// The path is adaptive: a row whose key does not fit the CTA table (table full / more than 8 probes) goes through the
// generic global path on the spot, and the host stops using this kernel when too many rows do that.
//
// Reference behaviour: AggOpenHashMap.putChunk (EX/operator/util/AggOpenHashMap.java:100-139) — same groups, same
// NULL rules; floating sums are accumulated in a different order (within the north_star's 1e-6 relative tolerance).
#pragma once

namespace {

constexpr int AF_THREADS = 512;
constexpr int AF_MAX_PROBES = 8;
constexpr int AF_MAX_USED = 8;
constexpr int AF_MAX_FV = 8;
constexpr int AF_STAGE_BYTES_PER_WARP = AF_MAX_USED * 32 * 8 + AF_MAX_USED * 32;
enum { C_FALLBACK = 2 };  // counters[2]: rows that bypassed the CTA table

struct SmemLayout {
    int32_t S;  // slots, power of two
    int32_t off_state;
    int32_t off_kv[GSQL_MAX_KEYS];
    int32_t off_kn[GSQL_MAX_KEYS];
    int32_t off_acc[GSQL_MAX_AGGS];
    int32_t off_cnt[GSQL_MAX_AGGS];  // AVG row count, -1 when unused
    int32_t off_has[GSQL_MAX_AGGS];
    int32_t total;
    // every input column the kernel touches (keys, aggregate arguments, derived operands, filters): loaded once per
    // row with all loads in flight, staged in a warp-private shared-memory strip, then read by column index
    int32_t nused;
    int32_t used[AF_MAX_USED];
    int8_t colmap[GSQL_MAX_COLS];  // input column -> staging row, -1 = unused
    int32_t off_stage;             // AF_MAX_USED x 32 x 8 B values + AF_MAX_USED x 32 B null flags
    int32_t warp_bytes;            // table + staging strip of one warp
    int32_t nfv;                   // fp64 SUM / AVG aggregates reduced together in ONE peer loop (<= AF_MAX_FV)
    int32_t fv_agg[AF_MAX_FV];
    int8_t fused[GSQL_MAX_AGGS];   // 1 = this aggregate is one of fv_agg
};

__device__ __forceinline__ int smem_find_or_insert(char *sm, const SmemLayout &L, int nkeys, const int64_t (&kv)[GSQL_MAX_KEYS],
                                                   const bool (&kn)[GSQL_MAX_KEYS], unsigned long long d) {
    if (nkeys == 0) return 0;
    int *state = reinterpret_cast<int *>(sm + L.off_state);
    int s = (int)(gsql_fmix64(d) & (unsigned long long)(L.S - 1));
    int probes = 0;
    while (probes < AF_MAX_PROBES) {
        int st = *reinterpret_cast<volatile int *>(&state[s]);
        if (st == 2) {
            bool eq = true;
            for (int c = 0; c < nkeys && eq; c++) {
                bool n = *reinterpret_cast<volatile uint8_t *>(sm + L.off_kn[c] + s) != 0;
                long long v = *reinterpret_cast<volatile long long *>(sm + L.off_kv[c] + (size_t)s * 8);
                if (n != kn[c] || (!n && v != kv[c])) eq = false;
            }
            if (eq) return s;
            s = (s + 1) & (L.S - 1);
            probes++;
        } else if (st == 0) {
            if (atomicCAS(&state[s], 0, 1) == 0) {
                for (int c = 0; c < nkeys; c++) {
                    *reinterpret_cast<long long *>(sm + L.off_kv[c] + (size_t)s * 8) = kv[c];
                    *reinterpret_cast<uint8_t *>(sm + L.off_kn[c] + s) = kn[c] ? 1 : 0;
                }
                __threadfence_block();
                *reinterpret_cast<volatile int *>(&state[s]) = 2;
                return s;
            }
        } else {
            __nanosleep(10);  // another lane is publishing this slot
        }
    }
    return -1;
}

// Sum of `v` over the lanes of `peers` (every lane of the warp calls this; each gets the sum of ITS peer group).
__device__ __forceinline__ double peer_sum_f64(double v, unsigned peers) {
    double s = 0.0;
    unsigned rem = peers;
    while (__any_sync(0xffffffffu, rem != 0)) {
        int src = rem ? __ffs(rem) - 1 : 0;
        double x = __shfl_sync(0xffffffffu, v, src);
        if (rem) {
            s += x;
            rem &= rem - 1;
        }
    }
    return s;
}
// Fused form: NV values reduced over the same peer groups with one pass over the peer bits.
template <int NV>
__device__ __forceinline__ void peer_sum_f64_multi(const double (&v)[NV], int nv, unsigned peers, double (&out)[NV]) {
#pragma unroll
    for (int j = 0; j < NV; j++) out[j] = 0.0;
    unsigned rem = peers;
    while (__any_sync(0xffffffffu, rem != 0)) {
        const int src = rem ? __ffs(rem) - 1 : 0;
        const bool take = rem != 0;
#pragma unroll
        for (int j = 0; j < NV; j++) {
            if (j < nv) {  // warp-uniform
                double x = __shfl_sync(0xffffffffu, v[j], src);
                if (take) out[j] += x;
            }
        }
        rem &= rem - 1;
    }
}
__device__ __forceinline__ long long peer_sum_i64(long long v, unsigned peers) {
    long long s = 0;
    unsigned rem = peers;
    while (__any_sync(0xffffffffu, rem != 0)) {
        int src = rem ? __ffs(rem) - 1 : 0;
        long long x = __shfl_sync(0xffffffffu, v, src);
        if (rem) {
            s = (long long)((unsigned long long)s + (unsigned long long)x);
            rem &= rem - 1;
        }
    }
    return s;
}
__device__ __forceinline__ long long peer_minmax_i64(long long v, unsigned peers, bool mx) {
    long long s = mx ? (long long)0x8000000000000000ULL : 0x7fffffffffffffffLL;
    unsigned rem = peers;
    while (__any_sync(0xffffffffu, rem != 0)) {
        int src = rem ? __ffs(rem) - 1 : 0;
        long long x = __shfl_sync(0xffffffffu, v, src);
        if (rem) {
            s = mx ? (x > s ? x : s) : (x < s ? x : s);
            rem &= rem - 1;
        }
    }
    return s;
}

__global__ void __launch_bounds__(AF_THREADS, 2) k_agg_smem(const __grid_constant__ AggParams P, const __grid_constant__ SmemLayout L) {
    extern __shared__ __align__(16) char sm_all[];
    const int lane = threadIdx.x & 31;
    const int warp_in_cta = threadIdx.x >> 5;
    char *sm = sm_all + (size_t)warp_in_cta * L.warp_bytes;  // this warp's table + staging strip
    // ---- init the warp table
    for (int i = lane; i < L.S; i += 32) {
        reinterpret_cast<int *>(sm + L.off_state)[i] = P.nkeys == 0 ? 2 : 0;
        for (int a = 0; a < P.naggs; a++) {
            long long init = P.agg[a].kind == GSQL_AGG_MIN ? 0x7fffffffffffffffLL : P.agg[a].kind == GSQL_AGG_MAX ? (long long)0x8000000000000000ULL : 0;
            reinterpret_cast<long long *>(sm + L.off_acc[a])[i] = init;
            if (L.off_cnt[a] >= 0) reinterpret_cast<long long *>(sm + L.off_cnt[a])[i] = 0;
            reinterpret_cast<uint8_t *>(sm + L.off_has[a])[i] = 0;
        }
    }
    __syncwarp();

    const int64_t warps_total = (int64_t)gridDim.x * (AF_THREADS / 32);
    const int64_t warp_id = (int64_t)blockIdx.x * (AF_THREADS / 32) + (threadIdx.x >> 5);
    unsigned long long *sval = reinterpret_cast<unsigned long long *>(sm + L.off_stage);
    uint8_t *snul = reinterpret_cast<uint8_t *>(sval + AF_MAX_USED * 32);
    // staged accessors (this lane's row): values are stored widened (INT32 sign-extended, FP64 as bits)
    auto s_null = [&](int col) -> bool { return snul[L.colmap[col] * 32 + lane] != 0; };
    auto s_raw = [&](int col) -> unsigned long long { return sval[L.colmap[col] * 32 + lane]; };
    auto s_f64 = [&](int col) -> double {
        unsigned long long v = s_raw(col);
        return P.in.c[col].type == GSQL_T_FP64 ? __longlong_as_double((long long)v) : (double)(long long)v;
    };
    auto s_i64 = [&](int col) -> long long {
        unsigned long long v = s_raw(col);
        return P.in.c[col].type == GSQL_T_FP64 ? (long long)__longlong_as_double((long long)v) : (long long)v;
    };
    auto v_null = [&](int col) -> bool {  // plain or derived column
        if (col < P.in.n) return s_null(col);
        const gsql_derived_col &d = P.derived[col - P.in.n];
        bool n = s_null(d.a) || s_null(d.b);
        if (d.kind == GSQL_EXPR_MUL_1MINUS_1PLUS) n = n || s_null(d.c);
        return n;
    };
    auto v_f64 = [&](int col) -> double {
        if (col < P.in.n) return s_f64(col);
        const gsql_derived_col &d = P.derived[col - P.in.n];
        double x = s_f64(d.a) * (1.0 - s_f64(d.b));
        if (d.kind == GSQL_EXPR_MUL_1MINUS_1PLUS) x = x * (1.0 + s_f64(d.c));
        return x;
    };
    auto v_i64 = [&](int col) -> long long { return col < P.in.n ? s_i64(col) : (long long)v_f64(col); };

    unsigned int fallback_rows = 0;
    for (int64_t b = warp_id * 32; b < P.rows; b += warps_total * 32) {
        const int64_t i = b + lane;
        const int64_t r = P.row0 + i;
        const bool inrange = i < P.rows;
        // ---- 1. every load of this row in flight at once, then staged
        {
            unsigned long long raw[AF_MAX_USED];
            uint8_t nul[AF_MAX_USED];
#pragma unroll
            for (int u = 0; u < AF_MAX_USED; u++) {
                raw[u] = 0;
                nul[u] = 0;
                if (u < L.nused && inrange) {
                    const DCol &col = P.in.c[L.used[u]];
                    if (col.type == GSQL_T_INT32) raw[u] = (unsigned long long)(long long)ld_stream_4(reinterpret_cast<const int *>(col.data) + r);
                    else raw[u] = (unsigned long long)ld_stream_8(reinterpret_cast<const long long *>(col.data) + r);
                    if (col.nulls) nul[u] = col.nulls[r];
                }
            }
#pragma unroll
            for (int u = 0; u < AF_MAX_USED; u++) {
                if (u < L.nused) {
                    sval[u * 32 + lane] = raw[u];
                    snul[u * 32 + lane] = nul[u];
                }
            }
        }
        // ---- 2. row filter, key, slot
        bool live = inrange;
        if (live && P.rf_op != GSQL_CMP_NONE) {
            if (s_null(P.rf_col)) live = false;
            else {
                long long v = s_i64(P.rf_col);
                switch (P.rf_op) {
                case GSQL_CMP_LE: live = v <= P.rf_value; break;
                case GSQL_CMP_LT: live = v < P.rf_value; break;
                case GSQL_CMP_GE: live = v >= P.rf_value; break;
                case GSQL_CMP_GT: live = v > P.rf_value; break;
                case GSQL_CMP_EQ: live = v == P.rf_value; break;
                default: live = v != P.rf_value; break;
                }
            }
        }
        int64_t kv[GSQL_MAX_KEYS];
        bool kn[GSQL_MAX_KEYS];
        unsigned long long d = 0;
        int slot = -2;
        if (live) {
            for (int c = 0; c < P.nkeys; c++) {  // canonical key image from the staged values (group key type = column type)
                const int col = P.keycol[c];
                kn[c] = s_null(col);
                long long v = (long long)s_raw(col);
                if (!kn[c] && P.in.c[col].type == GSQL_T_FP64) {
                    double x = __longlong_as_double(v);
                    if (x != x) v = 0x7ff8000000000000LL;
                    else if (x == 0.0) v = 0;
                }
                kv[c] = kn[c] ? 0 : v;
            }
            if (P.nkeys > 0) d = digest_of_keys(P, kv, kn);
            slot = smem_find_or_insert(sm, L, P.nkeys, kv, kn, d);
            if (slot == -1) {  // does not fit the CTA table: the generic path, right here
                fallback_rows++;
                int gid = find_group_kv(P, kv, kn, d);
                if (gid < 0) {
                    unsigned long long o = atomicAdd(&P.counters[C_OVERFLOW], 1ULL);
                    P.overflow_rows[o] = r;
                } else {
                    for (int a = 0; a < P.naggs; a++) accumulate(P, P.agg[a], gid, r);
                }
            }
        }
        const bool useful = slot >= 0;
        const unsigned peers = __match_any_sync(0xffffffffu, slot);
        const bool leader = useful && lane == __ffs(peers) - 1;
        // fp64 SUM / AVG arguments of all aggregates, reduced over the peer groups in one pass
        double fv[AF_MAX_FV], fsum[AF_MAX_FV];
        unsigned fokmask[AF_MAX_FV];
#pragma unroll
        for (int j = 0; j < AF_MAX_FV; j++) {
            fv[j] = 0.0;
            fokmask[j] = 0;
            if (j < L.nfv) {
                const AggDev &ag = P.agg[L.fv_agg[j]];
                bool ok = useful;
                if (ok && ag.filter_col >= 0)
                    if (P.in.c[ag.filter_col].type == GSQL_T_INT64 && !s_null(ag.filter_col) && s_i64(ag.filter_col) < 1) ok = false;
                if (ok && v_null(ag.cols[0])) ok = false;
                if (ok) fv[j] = v_f64(ag.cols[0]);
                fokmask[j] = __ballot_sync(0xffffffffu, ok);
            }
        }
        peer_sum_f64_multi<AF_MAX_FV>(fv, L.nfv, peers, fsum);
#pragma unroll
        for (int j = 0; j < AF_MAX_FV; j++) {
            if (j < L.nfv) {
                const int a = L.fv_agg[j];
                const unsigned long long cnt = __popc(peers & fokmask[j]);
                if (leader && cnt) {
                    reinterpret_cast<double *>(sm + L.off_acc[a])[slot] += fsum[j];
                    if (L.off_cnt[a] >= 0) reinterpret_cast<long long *>(sm + L.off_cnt[a])[slot] += (long long)cnt;
                    reinterpret_cast<uint8_t *>(sm + L.off_has[a])[slot] = 1;
                }
            }
        }
#pragma unroll 1
        for (int a = 0; a < P.naggs; a++) {
            const AggDev &ag = P.agg[a];
            if (L.fused[a]) continue;  // handled above
            bool ok = useful;
            if (ok && ag.filter_col >= 0) {
                if (P.in.c[ag.filter_col].type == GSQL_T_INT64 && !s_null(ag.filter_col) && s_i64(ag.filter_col) < 1) ok = false;
            }
            if (ok) {
                for (int q = 0; q < ag.ncols; q++)
                    if (v_null(ag.cols[q])) ok = false;  // COUNT: any NULL arg; others: the single argument
            }
            const unsigned okmask = __ballot_sync(0xffffffffu, ok);
            const unsigned long long cnt = __popc(peers & okmask);
            long long *acc = reinterpret_cast<long long *>(sm + L.off_acc[a]);
            switch (ag.kind) {
            case GSQL_AGG_COUNT_STAR:
            case GSQL_AGG_COUNT:
                if (leader && cnt) acc[slot] += (long long)cnt;
                break;
            case GSQL_AGG_SUM:
            case GSQL_AGG_AVG: {
                double v = ok ? v_f64(ag.cols[0]) : 0.0;
                double sum = peer_sum_f64(v, peers);
                if (leader && cnt) {
                    reinterpret_cast<double *>(acc)[slot] += sum;
                    if (L.off_cnt[a] >= 0) reinterpret_cast<long long *>(sm + L.off_cnt[a])[slot] += (long long)cnt;
                    reinterpret_cast<uint8_t *>(sm + L.off_has[a])[slot] = 1;
                }
                break;
            }
            case GSQL_AGG_SUM0: {
                long long v = ok ? v_i64(ag.cols[0]) : 0;
                long long sum = peer_sum_i64(v, peers);
                if (leader && cnt) acc[slot] = (long long)((unsigned long long)acc[slot] + (unsigned long long)sum);
                break;
            }
            default: {  // MIN / MAX on the order-preserving int64 image
                const bool mx = ag.kind == GSQL_AGG_MAX;
                long long ident = mx ? (long long)0x8000000000000000ULL : 0x7fffffffffffffffLL;
                long long v = ident;
                if (ok) v = ag.in_type == GSQL_T_FP64 ? dbl_sortable(v_f64(ag.cols[0]), mx) : v_i64(ag.cols[0]);
                long long m = peer_minmax_i64(v, peers, mx);
                if (leader && cnt) {
                    acc[slot] = mx ? (m > acc[slot] ? m : acc[slot]) : (m < acc[slot] ? m : acc[slot]);
                    reinterpret_cast<uint8_t *>(sm + L.off_has[a])[slot] = 1;
                }
            }
            }
        }
        __syncwarp();  // the next step's leaders (other lanes) read-modify-write the same accumulators
    }
    if (fallback_rows) atomicAdd(&P.counters[C_FALLBACK], (unsigned long long)fallback_rows);
    __syncwarp();
    // ---- merge this warp's partial groups into the global table
    for (int s = lane; s < L.S; s += 32) {
        if (reinterpret_cast<int *>(sm + L.off_state)[s] != 2) continue;
        int64_t kv[GSQL_MAX_KEYS];
        bool kn[GSQL_MAX_KEYS];
        for (int c = 0; c < P.nkeys; c++) {
            kv[c] = *reinterpret_cast<long long *>(sm + L.off_kv[c] + (size_t)s * 8);
            kn[c] = *reinterpret_cast<uint8_t *>(sm + L.off_kn[c] + s) != 0;
        }
        // a partial group without any contribution (all its rows filtered per aggregate) still has to exist as a group
        // the merge may exceed gcap by at most CTAs x S groups: covered by the arrays' slack (ignore_cap)
        int gid = P.nkeys == 0 ? 0 : find_group_kv(P, kv, kn, digest_of_keys(P, kv, kn), true);
        for (int a = 0; a < P.naggs; a++) {
            const AggDev &ag = P.agg[a];
            long long v = reinterpret_cast<long long *>(sm + L.off_acc[a])[s];
            bool has = reinterpret_cast<uint8_t *>(sm + L.off_has[a])[s] != 0;
            switch (ag.kind) {
            case GSQL_AGG_COUNT_STAR: case GSQL_AGG_COUNT: case GSQL_AGG_SUM0:
                if (v) atomicAdd(reinterpret_cast<unsigned long long *>(&ag.l[gid]), (unsigned long long)v);
                break;
            case GSQL_AGG_SUM:
                if (has) { atomicAdd(&ag.d[gid], __longlong_as_double(v)); ag.has[gid] = 1; }
                break;
            case GSQL_AGG_AVG:
                if (has) {
                    atomicAdd(&ag.d[gid], __longlong_as_double(v));
                    atomicAdd(reinterpret_cast<unsigned long long *>(&ag.l[gid]), (unsigned long long)reinterpret_cast<long long *>(sm + L.off_cnt[a])[s]);
                    ag.has[gid] = 1;
                }
                break;
            default:
                if (has) {
                    if (ag.kind == GSQL_AGG_MAX) atomicMax(reinterpret_cast<long long *>(&ag.l[gid]), v);
                    else atomicMin(reinterpret_cast<long long *>(&ag.l[gid]), v);
                    ag.has[gid] = 1;
                }
            }
        }
    }
}

}  // namespace

struct AggFast {
    bool eligible = false;  // shape supported by the shared-memory kernel
    bool enabled = false;   // still profitable (few rows bypass the CTA tables)
    SmemLayout L;
    FallbackRate rate;
};

// Decides eligibility and the shared-memory layout (host).
static void agg_fast_plan(AggFast *F, const gsql_agg_spec &spec, int nkeys, int naggs, const gsql_agg_call *aggs, const int32_t *in_type) {
    F->eligible = false;
    for (int a = 0; a < naggs; a++)
        if (aggs[a].kind == GSQL_AGG_SUM && in_type[a] != GSQL_T_FP64) return;  // exact 128-bit SUM(int) stays generic
    int per_slot = 4 + nkeys * 9;
    for (int a = 0; a < naggs; a++) per_slot += 8 + 1 + (aggs[a].kind == GSQL_AGG_AVG ? 8 : 0);
    int S = 1;
    if (nkeys > 0) S = per_slot <= 160 ? 32 : 16;  // slots of one WARP's table; more distinct keys bypass it (adaptive)
    SmemLayout &L = F->L;
    memset(&L, 0, sizeof(L));
    L.S = S;
    int off = 0;
    for (int a = 0; a < naggs; a++) { L.off_acc[a] = off; off += S * 8; }
    for (int a = 0; a < naggs; a++) {
        if (aggs[a].kind == GSQL_AGG_AVG) { L.off_cnt[a] = off; off += S * 8; }
        else L.off_cnt[a] = -1;
    }
    for (int c = 0; c < nkeys; c++) { L.off_kv[c] = off; off += S * 8; }
    L.off_state = off;
    off += S * 4;
    for (int c = 0; c < nkeys; c++) { L.off_kn[c] = off; off += S; }
    for (int a = 0; a < naggs; a++) { L.off_has[a] = off; off += S; }
    off = (off + 15) & ~15;
    // used input columns
    for (int c = 0; c < GSQL_MAX_COLS; c++) L.colmap[c] = -1;
    L.nused = 0;
    bool too_many = false;
    auto use = [&](int col) {
        if (col < 0) return;
        if (col >= spec.n_input_cols) {  // derived: its operands
            const gsql_derived_col &d = spec.derived[col - spec.n_input_cols];
            const int ops[3] = {d.a, d.b, d.kind == GSQL_EXPR_MUL_1MINUS_1PLUS ? d.c : -1};
            for (int q = 0; q < 3; q++)
                if (ops[q] >= 0 && L.colmap[ops[q]] < 0) {
                    if (L.nused == AF_MAX_USED) { too_many = true; return; }
                    L.colmap[ops[q]] = (int8_t)L.nused;
                    L.used[L.nused++] = ops[q];
                }
            return;
        }
        if (L.colmap[col] < 0) {
            if (L.nused == AF_MAX_USED) { too_many = true; return; }
            L.colmap[col] = (int8_t)L.nused;
            L.used[L.nused++] = col;
        }
    };
    for (int k = 0; k < nkeys; k++) use(spec.groups[k]);
    if (spec.row_filter_op != GSQL_CMP_NONE) use(spec.row_filter_col);
    for (int a = 0; a < naggs; a++) {
        use(aggs[a].filter_arg);
        for (int q = 0; q < aggs[a].ncols; q++) use(aggs[a].cols[q]);
    }
    if (too_many) return;
    L.nfv = 0;
    for (int a = 0; a < naggs; a++) {
        L.fused[a] = 0;
        if ((aggs[a].kind == GSQL_AGG_SUM || aggs[a].kind == GSQL_AGG_AVG) && L.nfv < AF_MAX_FV) {
            L.fused[a] = 1;
            L.fv_agg[L.nfv++] = a;
        }
    }
    L.off_stage = off;
    off += AF_STAGE_BYTES_PER_WARP;
    L.warp_bytes = (off + 15) & ~15;
    L.total = L.warp_bytes * (AF_THREADS / 32);
    F->eligible = true;
    F->enabled = true;
}
