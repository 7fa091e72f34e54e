// agg_reg.cuh — REGISTER accumulators for the NULL-free, very-low-cardinality group-by with fp64 sums (the TPC-H Q1
// shape as the plan hands it over: 2 integer keys, SUM / AVG over DOUBLE columns and fused derived expressions,
// COUNT(*), an integer row filter).  Included by agg.cu after agg_lane.cuh.
//
// Why another kernel: k_agg_lane keeps every accumulator in shared memory and decodes a plan per step, which makes it
// issue-bound at a few hundred thread instructions per row, far from the HBM roofline on config 3.  Here a thread owns RG_G x NSRC fp64 accumulators and RG_G counters in REGISTERS;
// a row costs its loads, one compare per group and NSRC predicated DADDs per group — ~100 thread instructions with
// NSRC x RG_G independent dependency chains.  The input columns of a tile reach shared memory through cp.async, one tile
// ahead of the accumulation (double buffer), so the HBM latency of the stream is never on a thread's critical path and no
// register holds a load in flight.  The (at most RG_G) group keys live in a per-block dictionary in shared memory that is
// only written when a new key shows up (the first tiles; warp-cooperative under a block lock, no block barrier in the row
// loop); a ninth key makes the row take the generic path on the spot (find_group_kv + L2 atomics), counted in
// C_FALLBACK so that the host stops choosing this kernel when that is common.  Everything that depends on the plan —
// the number of sums, the expression kind of each — is a template parameter or a warp-uniform branch on a
// __grid_constant__ descriptor; nothing is interpreted per row.
// When a block finishes, the register accumulators are reduced over the block (shuffles, then one shared-memory pass)
// and one thread per group folds them into the global table — exactly the merge of the other privatised kernels.
//
// Two kernels share that design.  k_agg_reg_pipe (further down; batches whose staged columns are 16-byte aligned — every
// cudaMalloc'd column): 512-row tiles brought in by cp.async.bulk, 3-4 stages with full / empty mbarriers, the faster
// of the two.  k_agg_reg (below; every other batch, e.g. views that start off a 16-byte boundary, which a bulk copy cannot
// read): 1024-row tiles in two buffers, staged by per-thread cp.async with no block barrier.  Both accumulate with
// one-hot DFMAs (rg_accumulate_onehot) and fall back to select-adds for rows that hold Inf / NaN.
//
// Reference behaviour: AggOpenHashMap.putChunk (EX/operator/util/AggOpenHashMap.java:100-139) with CountRow,
// Double2DoubleSum (LittleNum2DoubleSum.java:40-64) and SpecificType2DoubleAvgV2 (:51-84); same groups, sums added in a
// different order, counts bit-exact.  tests/test_agg_exact_gpu.py holds every sum to the exact value on dyadic inputs
// (exact in any order) and to the gamma_(n-1) * sum|x| rounding bound of any summation tree otherwise.
#pragma once

namespace {

constexpr int RG_THREADS = 256;
constexpr int RG_RPT = 4;       // rows per thread per tile
constexpr int RG_TILE = RG_THREADS * RG_RPT;
constexpr int RG_G = 8;         // groups a block can hold in registers (6 when there are 5-6 sums: 128 registers, two blocks per SM, no spills)
constexpr int RG_MAX_SRC = 6;   // distinct fp64 sums
constexpr int RG_MAX_USED = 8;  // distinct input columns a tile stages

struct RegSrc {
    int32_t kind;        // 0: column a; GSQL_EXPR_MUL_1MINUS: a*(1-b); GSQL_EXPR_MUL_1MINUS_1PLUS: a*(1-b)*(1+c)
    int32_t ua, ub, uc;  // staged-column slots
    int32_t oa, ob, oc;  // byte offsets of the operands' regions inside a tile buffer (host-flattened: with the source index a
    int32_t pad;         // compile-time constant after unrolling, these are direct constant-bank operands, no table walk)
};

struct RegPlan {
    int32_t nsrc, nkeys, nused, tile_bytes;
    RegSrc src[RG_MAX_SRC];
    int32_t used_col[RG_MAX_USED];   // input column of each staged slot
    int32_t used_off[RG_MAX_USED];   // byte offset of the slot's RG_TILE elements inside a tile buffer
    int32_t used_w[RG_MAX_USED];     // 4 or 8
    int32_t key_u[2];
    int32_t key_off[2], key_w[2];    // flattened copies for the row loop
    int32_t rf_u;                    // slot of the row-filter column, -1: no filter
    int32_t rf_off, rf_w, rf_neg;    // the filter as an interval test: pass = (lo <= x && x <= hi) != neg
    int64_t rf_lo, rf_hi;
    int32_t agg_src[GSQL_MAX_AGGS];  // per aggregate: the sum it reports, -1 for COUNT / COUNT(*)
    int32_t bulk_bytes;              // k_agg_reg_pipe: bytes one full tile brings in (sum of tile rows * used_w)
    int32_t stages;                  // k_agg_reg_pipe: tile buffers (3 or 4)
};

// Asynchronous copy (LDGSTS) of one tile's staged columns into `buf`: element (k * RG_THREADS + tid) of every column is
// copied — and later read back — by the same thread, so no block barrier is needed, only the thread's own wait_group.
__device__ __forceinline__ void rg_prefetch(const AggParams &P, const RegPlan &L, int64_t t0, unsigned char *buf) {
    const int tid = threadIdx.x;
    const int64_t left = P.rows - t0;
#pragma unroll 1
    for (int u = 0; u < L.nused; u++) {
        const DCol &c = P.in.c[L.used_col[u]];
        unsigned char *dst = buf + L.used_off[u];
        if (L.used_w[u] == 4) {
            const int *src = reinterpret_cast<const int *>(c.data) + P.row0 + t0;
#pragma unroll
            for (int k = 0; k < RG_RPT; k++) {
                const int i = k * RG_THREADS + tid;
                if (i < left) cp_async_4(dst + (size_t)i * 4, src + i);
            }
        } else {
            const long long *src = reinterpret_cast<const long long *>(c.data) + P.row0 + t0;
#pragma unroll
            for (int k = 0; k < RG_RPT; k++) {
                const int i = k * RG_THREADS + tid;
                if (i < left) cp_async_8(dst + (size_t)i * 8, src + i);
            }
        }
    }
    cp_async_commit();
}

// acc += v when gk == G0 — one ISETP and one predicated DADD (the `hit ? v : 0.0` form compiles to two FSELs and a DADD)
template <int G0>
__device__ __forceinline__ void rg_pred_add(double &acc, double v, int gk) {
    asm("{\n\t.reg .pred p;\n\tsetp.eq.s32 p, %2, %3;\n\t@p add.f64 %0, %0, %1;\n\t}" : "+d"(acc) : "d"(v), "r"(gk), "n"(G0));
}

__device__ __forceinline__ void reg_decode_key(const AggParams &P, const RegPlan &L, unsigned long long k, int64_t (&kv)[GSQL_MAX_KEYS], bool (&kn)[GSQL_MAX_KEYS]) {
    for (int c = 0; c < GSQL_MAX_KEYS; c++) { kv[c] = 0; kn[c] = false; }
    if (L.nkeys == 2) {
        kv[0] = (int64_t)(int32_t)(unsigned int)k;
        kv[1] = (int64_t)(int32_t)(unsigned int)(k >> 32);
    } else {
        kv[0] = L.key_w[0] == 4 ? (int64_t)(int32_t)(unsigned int)k : (int64_t)k;
    }
}

// Branch-free accumulate: G x NSRC select-and-add (ptxas turns the predicated fp64 add into two FSELs and a DADD).  The
// alternative — one divergent arm per group — was measured slower on the Q1 shape.
template <int NSRC, int G, int G0>
__device__ __forceinline__ void rg_accumulate(double (&acc)[G][NSRC], unsigned int (&cnt)[G], const double (&v)[NSRC], int gk) {
    if constexpr (G0 < G) {
        cnt[G0] += gk == G0 ? 1u : 0u;
#pragma unroll
        for (int j = 0; j < NSRC; j++) rg_pred_add<G0>(acc[G0][j], v[j], gk);
        rg_accumulate<NSRC, G, G0 + 1>(acc, cnt, v, gk);
    }
}

// One-hot accumulate: acc[g][j] = fma(v[j], m_g, acc[g][j]) with m_g = 1.0 for the row's group and 0.0 for the others —
// one DFMA per (group, sum) instead of a DADD and two FSELs.  Bit-identical to the select form for FINITE v: v * 1.0 is
// exact, v * 0.0 is a signed zero, and an accumulator that starts at +0.0 is never -0.0, so acc + (+-0.0) == acc.  A
// non-finite v (Inf * 0.0 = NaN would leak into the other groups) takes the select form: the caller tests the exponents.
template <int NSRC, int G>
__device__ __forceinline__ void rg_accumulate_onehot(double (&acc)[G][NSRC], unsigned int (&cnt)[G], const double (&v)[NSRC], int gk) {
#pragma unroll
    for (int g = 0; g < G; g++) {
        const bool hit = gk == g;
        cnt[g] += hit ? 1u : 0u;
        const double m = __hiloint2double(hit ? 0x3ff00000 : 0, 0);
#pragma unroll
        for (int j = 0; j < NSRC; j++) acc[g][j] = __fma_rn(v[j], m, acc[g][j]);
    }
}

template <int NSRC, int G>
__global__ void __launch_bounds__(RG_THREADS, 2) k_agg_reg(const __grid_constant__ AggParams P, const __grid_constant__ RegPlan L) {
    extern __shared__ __align__(16) unsigned char rg_smem[];  // two tile buffers
    __shared__ unsigned long long skey[G];
    __shared__ int s_ng, s_lock;
    __shared__ double red[RG_THREADS / 32][G][NSRC];
    __shared__ unsigned long long redc[RG_THREADS / 32][G];
    const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
    if (tid == 0) {
        s_ng = 0;
        s_lock = 0;
    }
    double acc[G][NSRC];
    unsigned int cnt[G];
#pragma unroll
    for (int g = 0; g < G; g++) {
        cnt[g] = 0;
#pragma unroll
        for (int j = 0; j < NSRC; j++) acc[g][j] = 0.0;
    }
    __syncthreads();
    unsigned long long fallback_rows = 0;
    const int64_t ntiles = (P.rows + RG_TILE - 1) / RG_TILE;
    int64_t tile = blockIdx.x;
    // every thread commits exactly one cp.async group per staged tile (an empty one past the last), so wait_group<1>
    // below waits for the current tile and leaves the next one in flight
    if (tile < ntiles) rg_prefetch(P, L, tile * RG_TILE, rg_smem);
    unsigned long long kk[G];  // this thread's copy of the block's key dictionary
    int ng = 0;
    for (int it = 0; tile < ntiles; tile += gridDim.x, it++) {
        const int64_t t0 = tile * RG_TILE;
        const int64_t next = tile + gridDim.x;
        const int st = it & 1;
        // the next tile's columns start their way from HBM before this tile is touched: the memory latency of the stream
        // is hidden behind the accumulation of a whole tile instead of being paid once per tile
        if (next < ntiles) rg_prefetch(P, L, next * RG_TILE, rg_smem + (size_t)(st ^ 1) * L.tile_bytes);
        else cp_async_commit();
        cp_async_wait<1>();
        const unsigned char *buf = rg_smem + (size_t)st * L.tile_bytes;
        const int64_t left = P.rows - t0;
        {  // refresh the register copy of the dictionary when another warp has added keys
            const int now = *reinterpret_cast<volatile int *>(&s_ng);
            if (now != ng) {
#pragma unroll
                for (int g = 0; g < G; g++)
                    if (g < now) kk[g] = *reinterpret_cast<volatile unsigned long long *>(&skey[g]);
                ng = now;
            }
        }
#pragma unroll 1
        for (int k = 0; k < RG_RPT; k++) {
            const int i = k * RG_THREADS + tid;
            bool pass = i < left;
            const unsigned char *row8 = buf + (size_t)i * 8, *row4 = buf + (size_t)i * 4;
            unsigned long long key = L.key_w[0] == 4 ? (unsigned long long)*reinterpret_cast<const unsigned int *>(row4 + L.key_off[0])
                                                     : *reinterpret_cast<const unsigned long long *>(row8 + L.key_off[0]);
            if (L.nkeys == 2) key |= (unsigned long long)*reinterpret_cast<const unsigned int *>(row4 + L.key_off[1]) << 32;
            if (L.rf_u >= 0) {  // fused scan-side predicate as an interval test (NULL-free column: checked by the plan)
                const long long x = L.rf_w == 4 ? (long long)*reinterpret_cast<const int *>(row4 + L.rf_off) : *reinterpret_cast<const long long *>(row8 + L.rf_off);
                pass = pass && ((x >= L.rf_lo && x <= L.rf_hi) != (L.rf_neg != 0));
            }
            int gid = -1;
#pragma unroll
            for (int g = 0; g < G; g++)
                if (g < ng && kk[g] == key) gid = g;
            // ---- a key this thread has not seen: add it to the block's dictionary (first tiles only); warp-cooperative, one
            // distinct key at a time, lane 0 takes the block's lock — no block barrier anywhere in the row loop
            unsigned need = __ballot_sync(0xffffffffu, pass && gid < 0);
            while (need) {
                const int leader = __ffs(need) - 1;
                const unsigned long long lk = __shfl_sync(0xffffffffu, key, leader);
                int got = -1;
                if (lane == 0) {
                    while (atomicCAS(&s_lock, 0, 1) != 0) {}
                    const int cur = *reinterpret_cast<volatile int *>(&s_ng);
                    for (int g = 0; g < cur; g++)
                        if (*reinterpret_cast<volatile unsigned long long *>(&skey[g]) == lk) got = g;
                    if (got < 0 && cur < G) {
                        *reinterpret_cast<volatile unsigned long long *>(&skey[cur]) = lk;
                        __threadfence_block();
                        *reinterpret_cast<volatile int *>(&s_ng) = cur + 1;
                        got = cur;
                    } else if (got < 0) {
                        got = -2;  // the dictionary is full: these rows take the generic path
                    }
                    __threadfence_block();
                    atomicExch(&s_lock, 0);
                }
                got = __shfl_sync(0xffffffffu, got, 0);
                if (pass && gid < 0 && key == lk) gid = got;
                if (got >= 0) {  // every lane learns the new entry
                    const int now = *reinterpret_cast<volatile int *>(&s_ng);
#pragma unroll
                    for (int g = 0; g < G; g++)
                        if (g < now) kk[g] = *reinterpret_cast<volatile unsigned long long *>(&skey[g]);
                    ng = now;
                }
                need = __ballot_sync(0xffffffffu, pass && gid == -1);
            }
            if (pass && gid == -2) {  // a ninth key: the generic path, right here
                fallback_rows++;
                int64_t kv[GSQL_MAX_KEYS];
                bool kn[GSQL_MAX_KEYS];
                reg_decode_key(P, L, key, kv, kn);
                const int64_t r = P.row0 + t0 + i;
                const int g2 = find_group_kv(P, kv, kn, digest_of_keys(P, kv, kn));
                if (g2 < 0) {
                    unsigned long long o = atomicAdd(&P.counters[C_OVERFLOW], 1ULL);
                    P.overflow_rows[o] = r;
                } else {
                    for (int a = 0; a < P.naggs; a++) accumulate(P, P.agg[a], g2, r);
                }
                pass = false;
            }
            // ---- accumulate: the row's values come out of shared memory (a dead row reads its own, in-buffer cell and is
            // masked by gk = -1), one compare per group, NSRC predicated adds
            double v[NSRC];
#pragma unroll
            for (int j = 0; j < NSRC; j++) {
                const RegSrc &sr = L.src[j];
                double x = *reinterpret_cast<const double *>(row8 + sr.oa);
                if (sr.kind != 0) {  // block-uniform
                    x = x * (1.0 - *reinterpret_cast<const double *>(row8 + sr.ob));
                    if (sr.kind == GSQL_EXPR_MUL_1MINUS_1PLUS) x = x * (1.0 + *reinterpret_cast<const double *>(row8 + sr.oc));
                }
                v[j] = x;
            }
            const int gk = pass ? gid : -1;
            int worst = 0;  // largest exponent field among the row's values: 0x7ff = Inf / NaN
#pragma unroll
            for (int j = 0; j < NSRC; j++) worst = max(worst, __double2hiint(v[j]) & 0x7ff00000);
            if (worst != 0x7ff00000) rg_accumulate_onehot<NSRC, G>(acc, cnt, v, gk);
            else rg_accumulate<NSRC, G, 0>(acc, cnt, v, gk);
        }
    }
    cp_async_wait<0>();
    if (fallback_rows) atomicAdd(&P.counters[C_FALLBACK], fallback_rows);
    // ---- merge: reduce over the warp with shuffles, over the block through shared memory, then one thread per group
    __syncthreads();
    const int ngf = s_ng;
#pragma unroll
    for (int g = 0; g < G; g++) {
        if (g >= ngf) break;
        unsigned int c = cnt[g];
#pragma unroll
        for (int d = 16; d > 0; d >>= 1) c += __shfl_xor_sync(0xffffffffu, c, d);
        if (lane == 0) redc[warp][g] = c;
#pragma unroll
        for (int j = 0; j < NSRC; j++) {
            const double sm = warp_sum_f64(acc[g][j]);
            if (lane == 0) red[warp][g][j] = sm;
        }
    }
    __syncthreads();
    if (tid < ngf) {
        const int g = tid;
        unsigned long long c = 0;
        double sums[NSRC];
#pragma unroll
        for (int j = 0; j < NSRC; j++) sums[j] = 0.0;
        for (int w = 0; w < RG_THREADS / 32; w++) {
            c += redc[w][g];
#pragma unroll
            for (int j = 0; j < NSRC; j++) sums[j] += red[w][g][j];
        }
        if (c) {  // (a key whose rows all failed the filter never entered the dictionary)
            int64_t kv[GSQL_MAX_KEYS];
            bool kn[GSQL_MAX_KEYS];
            reg_decode_key(P, L, skey[g], kv, kn);
            // the merge may exceed gcap by at most blocks x G groups: covered by the arrays' slack (ignore_cap)
            const int gl = find_group_kv(P, kv, kn, digest_of_keys(P, kv, kn), true);
            for (int a = 0; a < P.naggs; a++) {
                const AggDev &ag = P.agg[a];
                double sv = 0.0;
#pragma unroll
                for (int j = 0; j < NSRC; j++)
                    if (L.agg_src[a] == j) sv = sums[j];
                SState st;  // COUNT / COUNT(*): l = c; SUM: x = the sum; AVG: both
                st.x = __double_as_longlong(sv);
                st.l = (long long)c;
                st.has = 1;
                state_merge(ag, gl, st);
            }
        }
    }
}


// ================================================================================================ pipelined variant
// k_agg_reg_pipe: the same algorithm for batches whose staged columns are 16-byte aligned, rebuilt around what a
// profile of k_agg_reg showed once the loads were off the critical path (fixed-latency and short-scoreboard stalls, and
// the per-tile block barrier that bulk copies into two shared buffers need):
//   * S = 3-4 stages of 512-row tiles, a full / empty mbarrier pair per stage: a warp that finishes a tile releases it and
//     moves on — no block barrier; thread 0 refills a stage two tiles after it was consumed, so a straggling warp delays
//     nobody until it is a whole tile behind;
//   * the rows of a tile are handled in three unrolled passes — keys and filter for all rows, (rarely) the dictionary /
//     generic slow path, values and accumulate for all rows — so the shared-memory loads of the tile's rows are in flight
//     together instead of one row's dependent chain after the other;
//   * shared memory is addressed with explicit 32-bit addresses computed once per tile (ld.shared), not through generic
//     pointers re-derived per row (S2UR SR_CgaCtaId + ULEA + LDC in the old SASS).
// The ragged last tile is loaded synchronously by its owner block after the pipeline has drained.
constexpr int RGP_THREADS = 256;
constexpr int RGP_RPT = 2;
constexpr int RGP_TILE = RGP_THREADS * RGP_RPT;  // 512 rows
constexpr int RGP_MAX_STAGES = 4;

// (memory clobber: the compiler keeps them after the mbarrier wait / the tail's plain stores; ptxas still schedules the
// resulting LDS freely among the arithmetic)
__device__ __forceinline__ double rg_lds_f64(uint32_t a) {
    double v;
    asm volatile("ld.shared.f64 %0, [%1];" : "=d"(v) : "r"(a) : "memory");
    return v;
}
__device__ __forceinline__ unsigned long long rg_lds_u64(uint32_t a) {
    unsigned long long v;
    asm volatile("ld.shared.u64 %0, [%1];" : "=l"(v) : "r"(a) : "memory");
    return v;
}
__device__ __forceinline__ unsigned int rg_lds_u32(uint32_t a) {
    unsigned int v;
    asm volatile("ld.shared.u32 %0, [%1];" : "=r"(v) : "r"(a) : "memory");
    return v;
}

// A row whose key found no place in the block's dictionary: the generic table, right here (cold).
__device__ __noinline__ void rg_fallback_row(const AggParams &P, const RegPlan &L, unsigned long long key, int64_t r) {
    int64_t kv[GSQL_MAX_KEYS];
    bool kn[GSQL_MAX_KEYS];
    reg_decode_key(P, L, key, kv, kn);
    const int g2 = find_group_kv(P, kv, kn, digest_of_keys(P, kv, kn));
    if (g2 < 0) {
        unsigned long long o = atomicAdd(&P.counters[C_OVERFLOW], 1ULL);
        P.overflow_rows[o] = r;
    } else {
        for (int a = 0; a < P.naggs; a++) accumulate(P, P.agg[a], g2, r);
    }
}

// Warp-cooperative insertion of the keys this warp has not seen (same protocol as in k_agg_reg: one distinct key at a
// time, lane 0 takes the block's lock).  Every lane of the warp must call it.  gid: -1 unknown -> group index, or -2 when
// the dictionary is full.
template <int G>
__device__ __forceinline__ void rg_dict_insert(bool pass, int &gid, unsigned long long key, unsigned long long (&kk)[G], int &ng,
                                               unsigned long long *skey, int *s_ng, int *s_lock, int lane) {
    unsigned need = __ballot_sync(0xffffffffu, pass && gid < 0);
    while (need) {
        const int leader = __ffs(need) - 1;
        const unsigned long long lk = __shfl_sync(0xffffffffu, key, leader);
        int got = -1;
        if (lane == 0) {
            while (atomicCAS(s_lock, 0, 1) != 0) {}
            const int cur = *reinterpret_cast<volatile int *>(s_ng);
            for (int g = 0; g < cur; g++)
                if (*reinterpret_cast<volatile unsigned long long *>(&skey[g]) == lk) got = g;
            if (got < 0 && cur < G) {
                *reinterpret_cast<volatile unsigned long long *>(&skey[cur]) = lk;
                __threadfence_block();
                *reinterpret_cast<volatile int *>(s_ng) = cur + 1;
                got = cur;
            } else if (got < 0) {
                got = -2;
            }
            __threadfence_block();
            atomicExch(s_lock, 0);
        }
        got = __shfl_sync(0xffffffffu, got, 0);
        if (pass && gid < 0 && key == lk) gid = got;
        if (got >= 0) {
            const int now = *reinterpret_cast<volatile int *>(s_ng);
#pragma unroll
            for (int g = 0; g < G; g++)
                if (g < now) kk[g] = *reinterpret_cast<volatile unsigned long long *>(&skey[g]);
            ng = now;
        }
        need = __ballot_sync(0xffffffffu, pass && gid == -1);
    }
}

template <int NSRC, int G>
__global__ void __launch_bounds__(RGP_THREADS, 2) k_agg_reg_pipe(const __grid_constant__ AggParams P, const __grid_constant__ RegPlan L) {
    extern __shared__ __align__(128) unsigned char rg_smem[];  // L.stages tile buffers
    __shared__ unsigned long long skey[G];
    __shared__ int s_ng, s_lock;
    __shared__ double red[RGP_THREADS / 32][G][NSRC];
    __shared__ unsigned long long redc[RGP_THREADS / 32][G];
    __shared__ __align__(8) unsigned long long bar_full[RGP_MAX_STAGES], bar_empty[RGP_MAX_STAGES];
    const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
    const int S = L.stages, D = S - 2;  // prefetch distance: a stage is refilled two tiles after it was consumed
    if (tid == 0) {
        s_ng = 0;
        s_lock = 0;
        for (int s = 0; s < S; s++) {
            mbar_init(&bar_full[s], 1);
            mbar_init(&bar_empty[s], RGP_THREADS / 32);
        }
        asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
    }
    // Issuing a bulk copy is slow for the issuing thread (one thread issuing a tile's 7 copies made its warp the block's
    // straggler), so the work is spread: lane 0 of warp u copies staged column u, thread 0
    // also arms the tile's barrier.  (A complete_tx that lands before the expect_tx is legal: the phase cannot complete
    // before that arrival.)
    const bool issuer = lane == 0 && warp < L.nused;
    const unsigned char *src_next = nullptr;  // issuer: this block's next tile of its column
    uint32_t col_bytes = 0, dst_off = 0;
    uint64_t src_stride = 0, pol_stream = 0;
    if (issuer) {
        const DCol &c = P.in.c[L.used_col[warp]];
        const uint32_t w = (uint32_t)L.used_w[warp];
        col_bytes = RGP_TILE * w;
        dst_off = (uint32_t)L.used_off[warp];
        src_next = reinterpret_cast<const unsigned char *>(c.data) + (size_t)P.row0 * w + (size_t)blockIdx.x * col_bytes;
        src_stride = (uint64_t)gridDim.x * col_bytes;
        pol_stream = l2_policy_evict_first();
    }
    double acc[G][NSRC];
    unsigned int cnt[G];
#pragma unroll
    for (int g = 0; g < G; g++) {
        cnt[g] = 0;
#pragma unroll
        for (int j = 0; j < NSRC; j++) acc[g][j] = 0.0;
    }
    __syncthreads();
    unsigned long long fallback_rows = 0;
    unsigned long long kk[G];  // this thread's copy of the block's key dictionary
    int ng = 0;
    const int64_t nfull = P.rows / RGP_TILE;  // full tiles of the batch; tile j of this block is blockIdx.x + j * gridDim.x
    const int mine = nfull > blockIdx.x ? (int)((nfull - blockIdx.x + gridDim.x - 1) / gridDim.x) : 0;
    const uint32_t smem0 = smem_u32(rg_smem), full_a = smem_u32(bar_full), empty_a = smem_u32(bar_empty), sng_a = smem_u32(&s_ng);
    const uint32_t tile_bytes = (uint32_t)L.tile_bytes;
    auto issue = [&](int stage) {  // issuer threads only; tiles are issued in this block's tile order
        if (tid == 0) mbar_expect_tx(full_a + 8u * stage, (uint32_t)L.bulk_bytes);
        tma_load_1d(smem0 + (uint32_t)stage * tile_bytes + dst_off, src_next, col_bytes, full_a + 8u * stage, pol_stream);
        src_next += src_stride;
    };

    // one tile's rows: keys + filter, slow path when some key is new, values + accumulate.  `a8` / `a4` are the shared
    // addresses of this thread's first row in a region of 8- / 4-byte cells; row k sits RGP_THREADS cells further.
    auto consume = [&](uint32_t base, int64_t t0, int left) {
        const uint32_t a8 = base + (uint32_t)tid * 8u, a4 = base + (uint32_t)tid * 4u;
        {  // refresh the register copy of the dictionary when another warp has added keys
            const int now = (int)rg_lds_u32(sng_a);
            if (now != ng) {
#pragma unroll
                for (int g = 0; g < G; g++)
                    if (g < now) kk[g] = *reinterpret_cast<volatile unsigned long long *>(&skey[g]);
                ng = now;
            }
        }
        unsigned long long key[RGP_RPT];
        bool pass[RGP_RPT];
        int gid[RGP_RPT];
        bool unknown = false;
#pragma unroll
        for (int k = 0; k < RGP_RPT; k++) {
            const uint32_t o8 = (uint32_t)k * RGP_THREADS * 8u, o4 = (uint32_t)k * RGP_THREADS * 4u;
            pass[k] = k * RGP_THREADS + tid < left;
            key[k] = L.key_w[0] == 4 ? (unsigned long long)rg_lds_u32(a4 + (uint32_t)L.key_off[0] + o4) : rg_lds_u64(a8 + (uint32_t)L.key_off[0] + o8);
            if (L.nkeys == 2) key[k] |= (unsigned long long)rg_lds_u32(a4 + (uint32_t)L.key_off[1] + o4) << 32;
            if (L.rf_u >= 0) {
                const long long x = L.rf_w == 4 ? (long long)(int)rg_lds_u32(a4 + (uint32_t)L.rf_off + o4) : (long long)rg_lds_u64(a8 + (uint32_t)L.rf_off + o8);
                pass[k] = pass[k] && ((x >= L.rf_lo && x <= L.rf_hi) != (L.rf_neg != 0));
            }
            gid[k] = -1;
#pragma unroll
            for (int g = 0; g < G; g++)
                if (g < ng && kk[g] == key[k]) gid[k] = g;
            unknown = unknown || (pass[k] && gid[k] < 0);
        }
        if (__any_sync(0xffffffffu, unknown)) {  // first tiles only (or a dictionary that is full)
#pragma unroll
            for (int k = 0; k < RGP_RPT; k++) {
                rg_dict_insert<G>(pass[k], gid[k], key[k], kk, ng, skey, &s_ng, &s_lock, lane);
                if (pass[k] && gid[k] == -2) {
                    fallback_rows++;
                    rg_fallback_row(P, L, key[k], P.row0 + t0 + k * RGP_THREADS + tid);
                    pass[k] = false;
                }
            }
        }
#pragma unroll
        for (int k = 0; k < RGP_RPT; k++) {
            const uint32_t o8 = (uint32_t)k * RGP_THREADS * 8u;
            double v[NSRC];
#pragma unroll
            for (int j = 0; j < NSRC; j++) {
                const RegSrc &sr = L.src[j];
                double x = rg_lds_f64(a8 + (uint32_t)sr.oa + o8);
                if (sr.kind != 0) {  // block-uniform
                    x = x * (1.0 - rg_lds_f64(a8 + (uint32_t)sr.ob + o8));
                    if (sr.kind == GSQL_EXPR_MUL_1MINUS_1PLUS) x = x * (1.0 + rg_lds_f64(a8 + (uint32_t)sr.oc + o8));
                }
                v[j] = x;
            }
            const int gk = pass[k] ? gid[k] : -1;
            int worst = 0;
#pragma unroll
            for (int j = 0; j < NSRC; j++) worst = max(worst, __double2hiint(v[j]) & 0x7ff00000);
            if (worst != 0x7ff00000) rg_accumulate_onehot<NSRC, G>(acc, cnt, v, gk);
            else rg_accumulate<NSRC, G, 0>(acc, cnt, v, gk);
        }
    };

    if (issuer) {  // prologue: the first D tiles
        for (int j = 0; j < D && j < mine; j++) issue(j);
    }
    int st = 0;            // stage of tile j
    uint32_t ph = 0;       // its parity: (j / S) & 1
    int pst = D;           // issuers: the stage tile j + D goes to, == (j - 2) mod S ...
    uint32_t pph = 1;      // ... and, from j = 2 on, the parity of that stage's release by tile j - 2: ((j - 2) / S) & 1
                           // (toggled at every wrap of pst; the first wrap, at j = 1, brings it to 0)
    int64_t t0 = (int64_t)blockIdx.x * RGP_TILE;
    const int64_t t_stride = (int64_t)gridDim.x * RGP_TILE;
    // the ragged last tile of the batch is one more iteration of its owner block: loaded with plain loads after the
    // pipeline has drained (one tile per batch at most)
    const int tail = (int)(P.rows - nfull * RGP_TILE);
    const int iters = mine + ((tail > 0 && (int64_t)blockIdx.x == nfull % gridDim.x) ? 1 : 0);
    for (int j = 0; j < iters; j++, t0 += t_stride) {
        const bool full = j < mine;
        if (full) {
            if (issuer && j + D < mine) {
                if (j >= 2) mbar_wait(empty_a + 8u * pst, pph);  // every warp has released tile j - 2
                issue(pst);
            }
            if (++pst == S) { pst = 0; pph ^= 1u; }
            mbar_wait(full_a + 8u * st, ph);
        } else {
            __syncthreads();  // every warp is done with every stage; nothing is in flight (all issued tiles were consumed)
            t0 = nfull * RGP_TILE;
            for (int u = 0; u < L.nused; u++) {
                const DCol &c = P.in.c[L.used_col[u]];
                unsigned char *dst = rg_smem + (size_t)st * L.tile_bytes + L.used_off[u];
#pragma unroll
                for (int k = 0; k < RGP_RPT; k++) {
                    const int i = k * RGP_THREADS + tid;
                    if (i < tail) {
                        if (L.used_w[u] == 4) reinterpret_cast<int *>(dst)[i] = reinterpret_cast<const int *>(c.data)[P.row0 + t0 + i];
                        else reinterpret_cast<long long *>(dst)[i] = reinterpret_cast<const long long *>(c.data)[P.row0 + t0 + i];
                    }
                }
            }
            __syncwarp();  // a thread reads only the cells it wrote
        }
        consume(smem0 + (uint32_t)st * tile_bytes, t0, full ? RGP_TILE : tail);
        if (full) {
            __syncwarp();
            if (lane == 0) mbar_arrive(empty_a + 8u * st);
            if (++st == S) { st = 0; ph ^= 1u; }
        }
    }
    if (fallback_rows) atomicAdd(&P.counters[C_FALLBACK], fallback_rows);
    // ---- merge (as in k_agg_reg): warp shuffles, then shared memory, then one thread per group into the global table
    __syncthreads();
    const int ngf = s_ng;
#pragma unroll
    for (int g = 0; g < G; g++) {
        if (g >= ngf) break;
        unsigned int c = cnt[g];
#pragma unroll
        for (int d = 16; d > 0; d >>= 1) c += __shfl_xor_sync(0xffffffffu, c, d);
        if (lane == 0) redc[warp][g] = c;
#pragma unroll
        for (int j = 0; j < NSRC; j++) {
            const double sm = warp_sum_f64(acc[g][j]);
            if (lane == 0) red[warp][g][j] = sm;
        }
    }
    __syncthreads();
    if (tid < ngf) {
        const int g = tid;
        unsigned long long c = 0;
        double sums[NSRC];
#pragma unroll
        for (int j = 0; j < NSRC; j++) sums[j] = 0.0;
        for (int w = 0; w < RGP_THREADS / 32; w++) {
            c += redc[w][g];
#pragma unroll
            for (int j = 0; j < NSRC; j++) sums[j] += red[w][g][j];
        }
        if (c) {
            int64_t kv[GSQL_MAX_KEYS];
            bool kn[GSQL_MAX_KEYS];
            reg_decode_key(P, L, skey[g], kv, kn);
            const int gl = find_group_kv(P, kv, kn, digest_of_keys(P, kv, kn), true);
            for (int a = 0; a < P.naggs; a++) {
                const AggDev &ag = P.agg[a];
                double sv = 0.0;
#pragma unroll
                for (int j = 0; j < NSRC; j++)
                    if (L.agg_src[a] == j) sv = sums[j];
                SState st;  // COUNT / COUNT(*): l = c; SUM: x = the sum; AVG: both
                st.x = __double_as_longlong(sv);
                st.l = (long long)c;
                st.has = 1;
                state_merge(ag, gl, st);
            }
        }
    }
}

}  // namespace

// Create-time check of everything that does not depend on the batch.
static void agg_reg_check(AggFront *F, const gsql_agg_spec &spec, int nkeys, int naggs, const gsql_agg_call *aggs, const int32_t *in_type) {
    *F = AggFront{};
    if (nkeys < 1 || nkeys > 2) return;
    for (int k = 0; k < nkeys; k++) {
        const int t = spec.input_types[spec.groups[k]];
        if (t == GSQL_T_FP64) return;
        if (nkeys == 2 && t != GSQL_T_INT32) return;  // two keys must share one 64-bit word
    }
    for (int a = 0; a < naggs; a++) {
        if (aggs[a].filter_arg >= 0) return;
        switch (aggs[a].kind) {
        case GSQL_AGG_COUNT_STAR: case GSQL_AGG_COUNT: break;
        case GSQL_AGG_SUM: case GSQL_AGG_AVG:
            if (in_type[a] != GSQL_T_FP64) return;
            if (aggs[a].cols[0] < spec.n_input_cols && spec.input_types[aggs[a].cols[0]] != GSQL_T_FP64) return;
            break;
        default: return;
        }
    }
    if (spec.expected_groups > 4096) return;  // the planner expects far more groups than a block's registers hold
    F->shape_ok = F->enabled = true;
}

// Per-batch plan (NULL buffers are a property of the batch).  false = this batch takes another kernel.
static bool agg_reg_plan(RegPlan *Lp, const gsql_agg_spec &spec, int nkeys, int naggs, const gsql_agg_call *aggs, const DColSet &in, int tile_rows = RG_TILE) {
    RegPlan &L = *Lp;
    memset(&L, 0, sizeof(L));
    L.nkeys = nkeys;
    L.rf_u = -1;
    auto has_nulls = [&](int col) { return in.c[col].nulls != nullptr; };
    bool too_many = false;
    auto slot_of = [&](int col) -> int {  // staged slot of an input column
        for (int u = 0; u < L.nused; u++)
            if (L.used_col[u] == col) return u;
        if (L.nused == RG_MAX_USED) { too_many = true; return 0; }
        L.used_col[L.nused] = col;
        L.used_w[L.nused] = in.c[col].type == GSQL_T_INT32 ? 4 : 8;
        return L.nused++;
    };
    for (int k = 0; k < nkeys; k++) {
        if (has_nulls(spec.groups[k])) return false;
        L.key_u[k] = slot_of(spec.groups[k]);
    }
    if (spec.row_filter_op != GSQL_CMP_NONE) {
        if (has_nulls(spec.row_filter_col)) return false;
        L.rf_u = slot_of(spec.row_filter_col);
    }
    for (int a = 0; a < naggs; a++) {
        L.agg_src[a] = -1;
        const gsql_agg_call &c = aggs[a];
        if (c.kind == GSQL_AGG_COUNT) {  // COUNT(x...) == COUNT(*) exactly when no argument can be NULL
            for (int q = 0; q < c.ncols; q++) {
                const int col = c.cols[q];
                if (col < spec.n_input_cols) { if (has_nulls(col)) return false; }
                else {
                    const gsql_derived_col &d = spec.derived[col - spec.n_input_cols];
                    if (has_nulls(d.a) || has_nulls(d.b) || (d.kind == GSQL_EXPR_MUL_1MINUS_1PLUS && has_nulls(d.c))) return false;
                }
            }
            continue;
        }
        if (c.kind == GSQL_AGG_COUNT_STAR) continue;
        int kind = 0, oa, ob = 0, oc = 0;
        const int col = c.cols[0];
        if (col < spec.n_input_cols) {
            oa = col;
        } else {
            const gsql_derived_col &d = spec.derived[col - spec.n_input_cols];
            kind = d.kind; oa = d.a; ob = d.b; oc = d.kind == GSQL_EXPR_MUL_1MINUS_1PLUS ? d.c : d.b;
        }
        const int ops[3] = {oa, ob, oc};
        for (int q = 0; q < (kind == 0 ? 1 : 3); q++)
            if (has_nulls(ops[q]) || in.c[ops[q]].type != GSQL_T_FP64) return false;
        RegSrc s;
        s.kind = kind;
        s.ua = slot_of(oa);
        s.ub = kind ? slot_of(ob) : 0;
        s.uc = kind == GSQL_EXPR_MUL_1MINUS_1PLUS ? slot_of(oc) : 0;
        int at = -1;
        for (int j = 0; j < L.nsrc; j++)
            if (L.src[j].kind == s.kind && L.src[j].ua == s.ua && L.src[j].ub == s.ub && L.src[j].uc == s.uc) at = j;
        if (at < 0) {
            if (L.nsrc == RG_MAX_SRC) return false;
            at = L.nsrc;
            L.src[L.nsrc++] = s;
        }
        L.agg_src[a] = at;
    }
    if (too_many || L.nsrc == 0) return false;  // (pure COUNT(*) shapes stay on the lane kernel)
    int off = 0;  // 8-byte columns first: every region keeps its natural alignment
    for (int pass = 0; pass < 2; pass++)
        for (int u = 0; u < L.nused; u++)
            if ((L.used_w[u] == 8) == (pass == 0)) {
                L.used_off[u] = off;
                off += tile_rows * L.used_w[u];
            }
    L.tile_bytes = (off + 15) & ~15;
    L.bulk_bytes = off;
    for (int j = 0; j < L.nsrc; j++) {
        L.src[j].oa = L.used_off[L.src[j].ua];
        L.src[j].ob = L.used_off[L.src[j].ub];
        L.src[j].oc = L.used_off[L.src[j].uc];
    }
    for (int k = 0; k < nkeys; k++) {
        L.key_off[k] = L.used_off[L.key_u[k]];
        L.key_w[k] = L.used_w[L.key_u[k]];
    }
    if (L.rf_u >= 0) {  // every comparison with a constant is an interval test on integers
        L.rf_off = L.used_off[L.rf_u];
        L.rf_w = L.used_w[L.rf_u];
        const int64_t v = spec.row_filter_value, mn = INT64_MIN, mx = INT64_MAX;
        L.rf_lo = mn; L.rf_hi = mx; L.rf_neg = 0;
        switch (spec.row_filter_op) {
        case GSQL_CMP_LE: L.rf_hi = v; break;
        case GSQL_CMP_LT: if (v == mn) { L.rf_lo = 1; L.rf_hi = 0; } else L.rf_hi = v - 1; break;
        case GSQL_CMP_GE: L.rf_lo = v; break;
        case GSQL_CMP_GT: if (v == mx) { L.rf_lo = 1; L.rf_hi = 0; } else L.rf_lo = v + 1; break;
        case GSQL_CMP_EQ: L.rf_lo = L.rf_hi = v; break;
        default: L.rf_lo = L.rf_hi = v; L.rf_neg = 1; break;
        }
    }
    return true;
}
