// agg.cu — GPU hash aggregation behind gsql_agg_* (drop-in for HashAggExec consume / buildConsume / nextChunk).
//
// Reference path replaced (EX/ = polardbx-executor/src/main/java/com/alibaba/polardbx/executor/):
//   EX/operator/HashAggExec.java:133-145 (consumeChunk), :158-162 (buildConsume)
//   EX/operator/util/AggOpenHashMap.java:100-139 (putChunk), :160-194 (buildChunks)
//   EX/operator/util/GroupOpenHashMap.java:142-187 (doInnerPutArray, rehash)
//   EX/calc/aggfunctions/{CountRow,Count,LittleNum2DoubleSum,SpecificType2DoubleAvgV2,LittleNum2DecimalSum,
//                         Long2LongSum0,Int2IntMax,...}.java (accumulate / writeResultTo)
//
// Layout: one open-addressing table of 16-byte slots {digest, dense group id} in HBM (load <= 0.5); group
// keys and every accumulator are columnar arrays indexed by group id, updated with native L2 atomics
// (int64 add, fp64 add, int64 min/max on an order-preserving transform).  SUM(int|bigint) is exact 128-bit
// (lo/hi with carry), which equals the reference's long-with-overflow-escape-to-DECIMAL result.
// Two adaptive specialisations sit in front of the generic kernel: lane-private shared-memory accumulators for a
// handful of groups (agg_lane.cuh, the TPC-H Q1 shape) and warp-private shared-memory tables for tens of groups
// (agg_fast.cuh); rows whose key does not fit their small tables take the generic path inside the same kernel.
#include <algorithm>
#include <type_traits>

#include <cooperative_groups.h>
#include <cub/device/device_scan.cuh>

#include "common.cuh"

namespace {

constexpr unsigned long long DIGEST_EMPTY = 0x8000000000000000ULL;
constexpr int GID_PENDING = -1;
enum { C_NGROUPS = 0, C_OVERFLOW = 1, /* 2 = C_FALLBACK (agg_fast.cuh) */ C_FATAL = 3, C_COUNT = 4 };

struct __align__(16) ASlot {
    unsigned long long digest;
    int gid;
    unsigned int hasmask;  // hint, bit a: "aggregate a's state of this group is known to be non-NULL" (has[gid] == 1); 0 is always safe
};

// What the probe learned besides the group id: the slot and the hint it carried.  With it the per-row work on the table
// is one 16-byte slot read and the reductions — the separate reads of the group id and of every aggregate's `has` byte
// (two of the four L2 transactions per row on the C5 share) only happen until the hint is set.
struct SlotHint {
    ASlot *sl;
    unsigned int mask;
};

struct AggDev {  // device view of one aggregator's state
    int32_t kind, in_type, ncols, filter_col;
    int32_t cols[4];
    int64_t *l;      // count | int64 sum0 | min/max (sortable) | SUM(int) low word | FIRST_VALUE: FvCell per group
    int64_t *hi;     // SUM(int) high word | FIRST_VALUE (gsql_agg): one FvCell, the first non-NULL row of group 0
    double *d;       // fp64 sum
    uint8_t *has;    // "state is not NULL"
};

struct AggParams {
    DColSet in;
    KeySet keys;
    int32_t nkeys, naggs, exact, pad;
    ASlot *slots;
    uint64_t nslots;
    int64_t *gkey[GSQL_MAX_KEYS];  // group keys by gid (int widened / canonical double bits)
    uint8_t *gnull[GSQL_MAX_KEYS];
    AggDev agg[GSQL_MAX_AGGS];
    unsigned long long *counters;  // [C_NGROUPS], [C_OVERFLOW]
    int64_t *overflow_rows;        // row indices that found the table full
    const int64_t *row_list;       // non-null: process these rows (overflow re-run) instead of [row0, row0+rows)
    int64_t row0, rows;
    int64_t gcap;                  // groups the arrays can hold before a grow (a slack margin sits above it)
    int64_t garr;                  // hard capacity of the by-gid arrays (gcap + slack): a gid beyond it is never stored
    int32_t n_derived, rf_col, rf_op, pad2;
    int32_t keycol[GSQL_MAX_KEYS];  // input column index of each group key
    int64_t rf_value;
    gsql_derived_col derived[GSQL_MAX_DERIVED];
    unsigned long long fv_tag0;  // FIRST_VALUE: this consume call's ordinal, in place in the row tag (FV_ORD_SHIFT)
};

// FIRST_VALUE state: the (tag, value) of the earliest row seen, tag = ordinal | position | NULL bit (gsql_gpu.h).  The two
// words change together through a 16-byte CAS, so a reader never pairs one row's tag with another's value.
struct __align__(16) FvCell {
    unsigned long long tag;
    long long val;  // INT32 sign-extended, INT64, or FP64 bits
};
constexpr unsigned long long FV_EMPTY = ~0ULL;  // no row yet; its NULL bit is set, so an empty cell reads as NULL
constexpr int FV_POS_BITS = 36, FV_ORD_SHIFT = FV_POS_BITS + 1;
constexpr int64_t FV_MAX_ORDINAL = (1LL << (64 - FV_ORD_SHIFT)) - 2;  // all-ones ordinal is left to FV_EMPTY

// Lowers *p to (tag, val) when tag is smaller.  Tags only ever fall, and the read's tag half is one 8-byte word, so a
// stale or torn read shows a tag at least the current one: stopping on it is safe, and anything else is settled by the CAS.
// Most rows stop after the read: an earlier row has already set the cell.
__device__ __forceinline__ void fv_min(FvCell *p, unsigned long long tag, long long val) {
    const longlong2 w = __ldcg(reinterpret_cast<const longlong2 *>(p));
    FvCell cur{(unsigned long long)w.x, w.y};
    while (tag < cur.tag) {
        const FvCell prev = atomicCAS(p, cur, FvCell{tag, val});
        if (prev.tag == cur.tag && prev.val == cur.val) return;
        cur = prev;
    }
}

// canonical 8-byte image of a key component; NULL has its own flag
__device__ __forceinline__ int64_t canon_key(const KeyVal &k, int utype) {
    if (k.is_null) return 0;
    if (utype == GSQL_T_FP64) {
        double v = __longlong_as_double(k.i);
        if (v != v) return 0x7ff8000000000000LL;
        if (v == 0.0) return 0;
    }
    return k.i;
}

// order-preserving map double -> int64 (so that atomicMin/atomicMax on int64 implement Math.min/Math.max incl.
// -0.0 < +0.0).  NaN must win both: it is mapped to the extreme of the respective direction.
__device__ __forceinline__ long long dbl_sortable(double v, bool for_max) {
    if (v != v) return for_max ? 0x7fffffffffffffffLL : (long long)0x8000000000000000ULL;
    long long b = __double_as_longlong(v);
    return b ^ ((b >> 63) & 0x7fffffffffffffffLL);
}
__host__ __device__ __forceinline__ double dbl_unsortable(long long s, bool for_max) {
    if (for_max && s == 0x7fffffffffffffffLL) return __builtin_nan("");
    if (!for_max && s == (long long)0x8000000000000000ULL) return __builtin_nan("");
    long long b = s ^ ((s >> 63) & 0x7fffffffffffffffLL);
    double d;
    memcpy(&d, &b, 8);
    return d;
}

#include "agg_state.cuh"

__device__ __forceinline__ bool in_null(const DCol &c, int64_t r) { return c.nulls != nullptr && c.nulls[r] != 0; }

// The key helpers below are templated on the number of group keys: NK = 1..3 unrolls their loops over kv[] / kn[] so
// that the arrays live in registers; NK = 0 is the dynamic form (P.nkeys at run time), which indexes the arrays in a
// rolled loop and therefore keeps them in LOCAL memory — an 80-byte stack frame per thread that, at 2048 threads per SM,
// does not fit L1, so that traffic alone reaches L2 and DRAM on every row.  The row loops are instantiated for NK = 1, 2, 3.
// Table digest of a canonical key image: the key itself for a single key column (exact), a 64-bit mix otherwise.
template <int NK = 0>
__device__ __forceinline__ unsigned long long digest_of_keys(const AggParams &P, const int64_t (&kv)[GSQL_MAX_KEYS], const bool (&kn)[GSQL_MAX_KEYS]) {
    if (P.exact) return (unsigned long long)kv[0];
    unsigned long long h = 0x243F6A8885A308D3ULL;
    if constexpr (NK > 0) {
#pragma unroll
        for (int c = 0; c < NK; c++)
            h = gsql_fmix64(h ^ (unsigned long long)kv[c]) + (kn[c] ? 0xD6E8FEB86659FD93ULL : 0x9E3779B97F4A7C15ULL) * (unsigned)(c + 1);
    } else {
#pragma unroll 1
        for (int c = 0; c < P.nkeys; c++)
            h = gsql_fmix64(h ^ (unsigned long long)kv[c]) + (kn[c] ? 0xD6E8FEB86659FD93ULL : 0x9E3779B97F4A7C15ULL) * (unsigned)(c + 1);
    }
    if (h == DIGEST_EMPTY) h ^= 1;
    return h;
}

// Canonical key image of input row r (values + NULL flags) and its table digest.
template <int NK = 0>
__device__ __forceinline__ unsigned long long load_group_key(const AggParams &P, int64_t r, int64_t (&kv)[GSQL_MAX_KEYS], bool (&kn)[GSQL_MAX_KEYS]) {
    if constexpr (NK > 0) {
#pragma unroll
        for (int c = 0; c < NK; c++) {
            KeyVal k = gsql_load_key(P.keys.c[c], r, P.keys.utype[c]);
            kn[c] = k.is_null;
            kv[c] = canon_key(k, P.keys.utype[c]);
        }
    } else {
#pragma unroll 1
        for (int c = 0; c < P.nkeys; c++) {
            KeyVal k = gsql_load_key(P.keys.c[c], r, P.keys.utype[c]);
            kn[c] = k.is_null;
            kv[c] = canon_key(k, P.keys.utype[c]);
        }
    }
    return digest_of_keys<NK>(P, kv, kn);
}

// Finds or creates the group with key (kv, kn) / digest d.  Returns gid >= 0, or -1 when the table is full.
template <int NK = 0>
__device__ __forceinline__ int find_group_kv(const AggParams &P, const int64_t (&kv)[GSQL_MAX_KEYS], const bool (&kn)[GSQL_MAX_KEYS],
                                             unsigned long long d, bool ignore_cap = false, SlotHint *hint = nullptr) {
    if (NK == 0 && P.nkeys == 0) return 0;
    uint64_t s;
    bool dedicated = false;
    if (P.exact) {
        if (kn[0]) { s = P.nslots + 1; dedicated = true; }          // NULL group key is an ordinary key (Block.java:136-145)
        else if (d == DIGEST_EMPTY) { s = P.nslots; dedicated = true; }
    }
    if (!dedicated) s = __umul64hi(gsql_fmix64(d), P.nslots);
    while (true) {
        ASlot *sl = &P.slots[s];
        // first look through the read-only path with an evict_last hint (the partition's slice of the table stays in L2 under the
        // evict-first input stream).  A stale EMPTY is harmless: the CAS below returns the real content; a digest never changes
        // once written, so a stale non-EMPTY value cannot exist.
        // (one 16-byte read: digest, group id and hint; a stale id — still PENDING — is re-read below)
        const int4 w = ld_keep_16(sl, l2_policy_evict_last());
        unsigned long long cur = ((unsigned long long)(unsigned int)w.y << 32) | (unsigned int)w.x;
        bool from_load = true;  // `cur` is what the read returned (not the result of a CAS that lost)
        bool mine = false;
        if (dedicated) {
            // dedicated slots are claimed through gid only: digest field carries a "claimed" mark
            unsigned long long prev = cur == DIGEST_EMPTY ? atomicCAS(&sl->digest, DIGEST_EMPTY, 1ULL) : cur;
            if (prev == DIGEST_EMPTY) mine = true;
            else if (cur == DIGEST_EMPTY) from_load = false;
        } else if (cur == DIGEST_EMPTY) {
            if (!ignore_cap && *reinterpret_cast<volatile unsigned long long *>(&P.counters[C_NGROUPS]) >= (unsigned long long)P.gcap) return -1;
            unsigned long long prev = atomicCAS(&sl->digest, DIGEST_EMPTY, d);
            if (prev == DIGEST_EMPTY) mine = true;
            else { cur = prev; from_load = false; }
        }
        if (mine) {  // first appearance: allocate the dense group id, publish keys, then the id
            // the lanes that create a group in the same step share ONE bump of the group counter (a first batch of millions
            // of new groups used to serialise on that single L2 address)
            cooperative_groups::coalesced_group cg = cooperative_groups::coalesced_threads();
            unsigned long long gbase = 0;
            if (cg.thread_rank() == 0) gbase = atomicAdd(&P.counters[C_NGROUPS], (unsigned long long)cg.size());
            gbase = cg.shfl(gbase, 0);
            int gid = (int)gbase + (int)cg.thread_rank();
            if ((int64_t)gid >= P.garr) {  // cannot happen while the host grows after every launch (slack covers one launch's merges):
                P.counters[C_FATAL] = 1;   // never write out of bounds — the host turns this into an error
                gid = (int)(P.garr - 1);
            } else if constexpr (NK > 0) {
#pragma unroll
                for (int c = 0; c < NK; c++) {
                    P.gkey[c][gid] = kv[c];
                    P.gnull[c][gid] = kn[c] ? 1 : 0;
                }
            } else {
                for (int c = 0; c < P.nkeys; c++) {
                    P.gkey[c][gid] = kv[c];
                    P.gnull[c][gid] = kn[c] ? 1 : 0;
                }
            }
            __threadfence();
            *reinterpret_cast<volatile int *>(&sl->gid) = gid;
            if (hint) { hint->sl = sl; hint->mask = 0; }
            return gid;
        }
        if (dedicated || cur == d) {
            int gid = from_load ? w.z : GID_PENDING;
            while (gid == GID_PENDING) {
                gid = *reinterpret_cast<volatile int *>(&sl->gid);
                if (gid == GID_PENDING) __nanosleep(20);
            }
            if (hint) { hint->sl = sl; hint->mask = from_load ? (unsigned int)w.w : 0u; }
            if (P.exact) return gid;
            __threadfence();
            bool eq = true;
            if constexpr (NK > 0) {
#pragma unroll
                for (int c = 0; c < NK; c++) {
                    if (eq) {
                        bool gn = *reinterpret_cast<volatile uint8_t *>(&P.gnull[c][gid]) != 0;
                        long long gv = *reinterpret_cast<volatile long long *>(&P.gkey[c][gid]);
                        if (gn != kn[c] || (!gn && gv != kv[c])) eq = false;
                    }
                }
            } else {
                for (int c = 0; c < P.nkeys && eq; c++) {
                    bool gn = *reinterpret_cast<volatile uint8_t *>(&P.gnull[c][gid]) != 0;
                    long long gv = *reinterpret_cast<volatile long long *>(&P.gkey[c][gid]);
                    if (gn != kn[c] || (!gn && gv != kv[c])) eq = false;
                }
            }
            if (eq) return gid;
        }
        if (++s == P.nslots) s = 0;
    }
}

template <int NK = 0>
__device__ __forceinline__ int find_group(const AggParams &P, int64_t r, SlotHint *hint = nullptr) {
    if (NK == 0 && P.nkeys == 0) return 0;
    int64_t kv[GSQL_MAX_KEYS];
    bool kn[GSQL_MAX_KEYS];
    unsigned long long d = load_group_key<NK>(P, r, kv, kn);
    return find_group_kv<NK>(P, kv, kn, d, false, hint);
}

__device__ __forceinline__ int64_t in_i64(const DCol &c, int64_t r) {  // streaming (evict-first) reads: every input value is used once
    if (c.type == GSQL_T_INT32) return __ldcs(reinterpret_cast<const int *>(c.data) + r);
    if (c.type == GSQL_T_INT64) return __ldcs(reinterpret_cast<const long long *>(c.data) + r);
    return (int64_t)__ldcs(reinterpret_cast<const double *>(c.data) + r);
}
__device__ __forceinline__ double in_f64(const DCol &c, int64_t r) {
    if (c.type == GSQL_T_FP64) return __ldcs(reinterpret_cast<const double *>(c.data) + r);
    if (c.type == GSQL_T_INT64) return (double)__ldcs(reinterpret_cast<const long long *>(c.data) + r);
    return (double)__ldcs(reinterpret_cast<const int *>(c.data) + r);
}

// Column `col` of row r as the aggregators see it: a plain input column, or a fused derived expression
// (VectorizedProjectExec replacement): NULL when any operand is NULL.
__device__ __forceinline__ bool val_null(const AggParams &P, int col, int64_t r) {
    if (col < P.in.n) return in_null(P.in.c[col], r);
    const gsql_derived_col &d = P.derived[col - P.in.n];
    bool n = in_null(P.in.c[d.a], r) || in_null(P.in.c[d.b], r);
    if (d.kind == GSQL_EXPR_MUL_1MINUS_1PLUS) n = n || in_null(P.in.c[d.c], r);
    return n;
}
__device__ __forceinline__ double val_f64(const AggParams &P, int col, int64_t r) {
    if (col < P.in.n) return in_f64(P.in.c[col], r);
    const gsql_derived_col &d = P.derived[col - P.in.n];
    double x = in_f64(P.in.c[d.a], r) * (1.0 - in_f64(P.in.c[d.b], r));
    if (d.kind == GSQL_EXPR_MUL_1MINUS_1PLUS) x = x * (1.0 + in_f64(P.in.c[d.c], r));
    return x;
}
__device__ __forceinline__ int64_t val_i64(const AggParams &P, int col, int64_t r) {
    if (col < P.in.n) return in_i64(P.in.c[col], r);
    return (int64_t)val_f64(P, col, r);
}
// the value's bits as FIRST_VALUE keeps them: INT32 sign-extended, INT64 and FP64 unchanged (no canonicalisation)
__device__ __forceinline__ long long in_bits(const DCol &c, int64_t r) {
    if (c.type == GSQL_T_INT32) return __ldcs(reinterpret_cast<const int *>(c.data) + r);
    return __ldcs(reinterpret_cast<const long long *>(c.data) + r);
}
// fused scan-side predicate (VectorizedFilterExec replacement); NULL never passes
__device__ __forceinline__ bool row_passes(const AggParams &P, int64_t r) {
    if (P.rf_op == GSQL_CMP_NONE) return true;
    const DCol &c = P.in.c[P.rf_col];
    if (in_null(c, r)) return false;
    int64_t v = in_i64(c, r);
    switch (P.rf_op) {
    case GSQL_CMP_LE: return v <= P.rf_value;
    case GSQL_CMP_LT: return v < P.rf_value;
    case GSQL_CMP_GE: return v >= P.rf_value;
    case GSQL_CMP_GT: return v > P.rf_value;
    case GSQL_CMP_EQ: return v == P.rf_value;
    default: return v != P.rf_value;
    }
}

// "This group's state of aggregate `aidx` is not NULL any more."  The slot's hint bit, once set, spares the row both the
// read of has[gid] and the store; until then: a read that hits L2 instead of a one-byte store per row, and one RED.OR.
__device__ __forceinline__ void mark_has(const AggDev &a, int gid, int aidx, SlotHint *h) {
    if (h != nullptr && aidx >= 0 && ((h->mask >> aidx) & 1u)) return;
    if (!ld_keep_u8(&a.has[gid], l2_policy_evict_last())) a.has[gid] = 1;
    if (h != nullptr && h->sl != nullptr && aidx >= 0) atomicOr(&h->sl->hasmask, 1u << aidx);
}

__device__ __forceinline__ void accumulate(const AggParams &P, const AggDev &a, int gid, int64_t r, int aidx = -1, SlotHint *h = nullptr) {
    if (a.filter_col >= 0) {  // AggOpenHashMap.java:114-131 — only Boolean / Long objects filter
        const DCol &f = P.in.c[a.filter_col];
        if (f.type == GSQL_T_INT64 && !in_null(f, r) && reinterpret_cast<const int64_t *>(f.data)[r] < 1) return;
    }
    switch (a.kind) {
    case GSQL_AGG_COUNT_STAR:
        red_add_u64_keep(reinterpret_cast<unsigned long long *>(&a.l[gid]), 1ULL, l2_policy_evict_last());
        return;
    case GSQL_AGG_COUNT:
        for (int i = 0; i < a.ncols; i++)
            if (val_null(P, a.cols[i], r)) return;
        atomicAdd(reinterpret_cast<unsigned long long *>(&a.l[gid]), 1ULL);
        return;
    default: break;
    }
    const int c = a.cols[0];
    if (val_null(P, c, r)) return;
    switch (a.kind) {
    case GSQL_AGG_SUM:
        if (a.in_type == GSQL_T_FP64) {
            red_add_f64_keep(&a.d[gid], val_f64(P, c, r), l2_policy_evict_last());
        } else {  // exact 128-bit: lo += v (carry out), hi += sign extension + carry
            long long v = val_i64(P, c, r);
            unsigned long long old = atomicAdd(reinterpret_cast<unsigned long long *>(&a.l[gid]), (unsigned long long)v);
            unsigned long long sum = old + (unsigned long long)v;
            long long carry = (sum < old ? 1 : 0) + (v < 0 ? -1 : 0);
            if (carry) atomicAdd(reinterpret_cast<unsigned long long *>(&a.hi[gid]), (unsigned long long)carry);
        }
        mark_has(a, gid, aidx, h);
        return;
    case GSQL_AGG_AVG:
        atomicAdd(&a.d[gid], val_f64(P, c, r));
        atomicAdd(reinterpret_cast<unsigned long long *>(&a.l[gid]), 1ULL);
        mark_has(a, gid, aidx, h);
        return;
    case GSQL_AGG_SUM0:
        atomicAdd(reinterpret_cast<unsigned long long *>(&a.l[gid]), (unsigned long long)val_i64(P, c, r));
        return;
    case GSQL_AGG_AVG_MERGE:  // (partial sum, partial count): the sum is NULL exactly when its count is 0
        atomicAdd(&a.d[gid], val_f64(P, c, r));
        if (!val_null(P, a.cols[1], r)) atomicAdd(reinterpret_cast<unsigned long long *>(&a.l[gid]), (unsigned long long)val_i64(P, a.cols[1], r));
        mark_has(a, gid, aidx, h);
        return;
    case GSQL_AGG_MIN:
    case GSQL_AGG_MAX: {
        bool mx = a.kind == GSQL_AGG_MAX;
        long long v = a.in_type == GSQL_T_FP64 ? dbl_sortable(val_f64(P, c, r), mx) : val_i64(P, c, r);
        if (mx) atomicMax(reinterpret_cast<long long *>(&a.l[gid]), v);
        else atomicMin(reinterpret_cast<long long *>(&a.l[gid]), v);
        mark_has(a, gid, aidx, h);
        return;
    }
    default: return;
    }
}

// FIRST_VALUE, in the generic row loop's FV instantiation only: the privatised kernels, which share accumulate(), are off for
// such specs, and the row loop without it keeps its registers.
// A NULL row counts as a first row too (InternalFirstValue.accumulate:96-108).
__device__ __forceinline__ void accumulate_first(const AggParams &P, const AggDev &a, int gid, int64_t r) {
    const int c = a.cols[0];
    const bool n = val_null(P, c, r);
    const long long v = n ? 0 : (c < P.in.n ? in_bits(P.in.c[c], r) : __double_as_longlong(val_f64(P, c, r)));
    const unsigned long long tag = P.fv_tag0 | ((unsigned long long)r << 1) | (n ? 1ULL : 0ULL);  // r: position as passed
    fv_min(reinterpret_cast<FvCell *>(a.l) + gid, tag, v);
    if (gid == 0 && !n) fv_min(reinterpret_cast<FvCell *>(a.hi), tag, v);  // the one-group rule's candidate
}

// The generic row loop.  Its trip count is warp-uniform and the warp is brought back together twice per row
// (__syncwarp): the probe of the table is divergent by nature, and without the explicit reconvergence the lanes drifted
// apart for good — the key and value loads of the next rows then execute with a fraction of the lanes active, each
// fetching its own 32-byte sector instead of sharing one per four rows.
template <int NK, bool FV>
__device__ __forceinline__ void agg_rows(const AggParams &P) {
    const int lane = threadIdx.x & 31;
    const int64_t stride = (int64_t)gridDim.x * blockDim.x;
    for (int64_t base = blockIdx.x * (int64_t)blockDim.x + (threadIdx.x - lane); base < P.rows; base += stride) {
        const int64_t i = base + lane;
        const bool live = i < P.rows;
        const int64_t r = live ? (P.row_list ? P.row_list[i] : P.row0 + i) : 0;
        const bool pass = live && row_passes(P, r);
        int gid = -1;
        SlotHint hint{nullptr, 0u};
        if (pass) gid = find_group<NK>(P, r, &hint);
        __syncwarp();  // the aggregates' input loads below are issued by the whole warp again: coalesced
        if (pass) {
            if (gid < 0) {
                unsigned long long o = atomicAdd(&P.counters[C_OVERFLOW], 1ULL);
                P.overflow_rows[o] = r;
            } else {
                for (int a = 0; a < P.naggs; a++) {
                    if (FV && P.agg[a].kind == GSQL_AGG_FIRST_VALUE) accumulate_first(P, P.agg[a], gid, r);
                    else accumulate(P, P.agg[a], gid, r, a, &hint);
                }
            }
        }
        __syncwarp();  // ... and so are the key loads of the next row
    }
}
template <int NK>
__global__ void __launch_bounds__(256) k_agg_consume(const __grid_constant__ AggParams P) { agg_rows<NK, false>(P); }
// specs with FIRST_VALUE: the 16-byte CAS loop's registers; at the default target the loop spilled
template <int NK>
__global__ void __launch_bounds__(256, 6) k_agg_consume_fv(const __grid_constant__ AggParams P) { agg_rows<NK, true>(P); }

// ---- pre-pass for tables beyond L2 (default; GSQL_AGG_PARTITION=0 disables): the batch is reordered by
// the high bits of the same hash that picks the table slot, so that k_agg_consume — which walks rows in index order —
// touches one L2-sized slice of the slot array at a time; dense group ids are handed out in first-appearance order,
// so the accumulators of a slice's groups are contiguous (and L2-resident) as well.  Same idea as the radix mode of
// the join (join_fast.cuh): an HBM-resident slot read costs a whole-line fetch, and an fp64 atomic on a line that misses
// L2 is many times slower than one on a resident line (tools/microbench.cu measures both).
struct APart {
    int32_t nparts, nblocks;
    int64_t chunk;  // rows per block
};
struct APartOut {
    void *data[GSQL_MAX_COLS];
    uint8_t *nulls[GSQL_MAX_COLS];
};

template <int NK>
__device__ __forceinline__ int agg_part_of(const AggParams &P, int64_t r, int nparts) {
    int64_t kv[GSQL_MAX_KEYS];
    bool kn[GSQL_MAX_KEYS];
    unsigned long long d = load_group_key<NK>(P, r, kv, kn);
    return (int)__umul64hi(gsql_fmix64(d), (uint64_t)nparts);  // slot = mulhi(fmix64(d), nslots): partition = slot range
}

template <int NK>
__global__ void __launch_bounds__(256) k_agg_part_hist(const __grid_constant__ AggParams P, APart G, int64_t *__restrict__ hist) {
    extern __shared__ unsigned int sh_part[];
    for (int i = threadIdx.x; i < G.nparts; i += 256) sh_part[i] = 0;
    __syncthreads();
    int64_t r0 = (int64_t)blockIdx.x * G.chunk;
    int64_t r1 = r0 + G.chunk < P.rows ? r0 + G.chunk : P.rows;
    for (int64_t r = r0 + threadIdx.x; r < r1; r += 256) atomicAdd(&sh_part[agg_part_of<NK>(P, r, G.nparts)], 1u);
    __syncthreads();
    for (int i = threadIdx.x; i < G.nparts; i += 256) hist[(int64_t)i * G.nblocks + blockIdx.x] = sh_part[i];
}

template <int NK>
__global__ void __launch_bounds__(256)
    k_agg_part_scatter(const __grid_constant__ AggParams P, APart G, const int64_t *__restrict__ offs, const __grid_constant__ APartOut O) {
    extern __shared__ unsigned long long cur_part[];
    for (int i = threadIdx.x; i < G.nparts; i += 256) cur_part[i] = (unsigned long long)offs[(int64_t)i * G.nblocks + blockIdx.x];
    __syncthreads();
    int64_t r0 = (int64_t)blockIdx.x * G.chunk;
    int64_t r1 = r0 + G.chunk < P.rows ? r0 + G.chunk : P.rows;
    for (int64_t base = r0; base < r1; base += 256) {
        int64_t r = base + threadIdx.x;
        bool live = r < r1;
        int p = live ? agg_part_of<NK>(P, r, G.nparts) : -1;
        unsigned peers = __match_any_sync(0xffffffffu, p);  // one shared-memory atomic per distinct partition per warp
        int lane = threadIdx.x & 31;
        int leader = __ffs(peers) - 1;
        unsigned long long basepos = 0;
        if (live && lane == leader) basepos = atomicAdd(&cur_part[p], (unsigned long long)__popc(peers));
        basepos = __shfl_sync(0xffffffffu, basepos, leader);
        if (!live) continue;
        int64_t pos = (int64_t)basepos + __popc(peers & ((1u << lane) - 1));
        for (int c = 0; c < P.in.n; c++) {
            const DCol &col = P.in.c[c];
            if (col.type == GSQL_T_INT32) reinterpret_cast<int32_t *>(O.data[c])[pos] = reinterpret_cast<const int32_t *>(col.data)[r];
            else reinterpret_cast<int64_t *>(O.data[c])[pos] = reinterpret_cast<const int64_t *>(col.data)[r];
            if (O.nulls[c]) O.nulls[c][pos] = col.nulls[r];
        }
    }
}

__global__ void __launch_bounds__(256) k_aslots_init(ASlot *slots, uint64_t n) {
    for (uint64_t i = blockIdx.x * (uint64_t)blockDim.x + threadIdx.x; i < n; i += (uint64_t)gridDim.x * blockDim.x) {
        int4 v;
        v.x = 0;
        v.y = (int)0x80000000;
        v.z = GID_PENDING;
        v.w = 0;
        reinterpret_cast<int4 *>(slots)[i] = v;
    }
}

__global__ void __launch_bounds__(256) k_fill_i64(int64_t *p, int64_t v, int64_t from, int64_t to) {
    for (int64_t i = from + blockIdx.x * (int64_t)blockDim.x + threadIdx.x; i < to; i += (int64_t)gridDim.x * blockDim.x) p[i] = v;
}

// re-insert groups [0, ngroups) into a fresh slot array after a grow (GroupOpenHashMap.rehash:171-187)
__global__ void __launch_bounds__(256) k_agg_rehash(const __grid_constant__ AggParams P, int64_t ngroups) {
    for (int64_t g = blockIdx.x * (int64_t)blockDim.x + threadIdx.x; g < ngroups; g += (int64_t)gridDim.x * blockDim.x) {
        unsigned long long d;
        uint64_t s;
        bool dedicated = false;
        if (P.exact) {
            d = (unsigned long long)P.gkey[0][g];
            if (P.gnull[0][g]) { s = P.nslots + 1; dedicated = true; }
            else if (d == DIGEST_EMPTY) { s = P.nslots; dedicated = true; }
        } else {
            unsigned long long h = 0x243F6A8885A308D3ULL;
            for (int c = 0; c < P.nkeys; c++) {
                bool n = P.gnull[c][g] != 0;
                h = gsql_fmix64(h ^ (unsigned long long)P.gkey[c][g]) + (n ? 0xD6E8FEB86659FD93ULL : 0x9E3779B97F4A7C15ULL) * (unsigned)(c + 1);
            }
            if (h == DIGEST_EMPTY) h ^= 1;
            d = h;
        }
        if (dedicated) {
            P.slots[s].digest = 1ULL;
            P.slots[s].gid = (int)g;
            continue;
        }
        s = __umul64hi(gsql_fmix64(d), P.nslots);
        while (atomicCAS(&P.slots[s].digest, DIGEST_EMPTY, d) != DIGEST_EMPTY)
            if (++s == P.nslots) s = 0;
        P.slots[s].gid = (int)g;
    }
}

struct FinalCol {
    void *data;
    uint8_t *nulls;
    int32_t type, pad;
};
struct FinalParams {
    int32_t nkeys, naggs;
    int64_t ngroups;
    const int64_t *gkey[GSQL_MAX_KEYS];
    const uint8_t *gnull[GSQL_MAX_KEYS];
    int32_t key_types[GSQL_MAX_KEYS];
    AggDev agg[GSQL_MAX_AGGS];
    FinalCol out[GSQL_MAX_COLS];
};

// writeResultTo per group, in group-id order (AggOpenHashMap.buildValueChunks:160-178)
__global__ void __launch_bounds__(256) k_agg_finalize(const __grid_constant__ FinalParams F) {
    for (int64_t g = blockIdx.x * (int64_t)blockDim.x + threadIdx.x; g < F.ngroups; g += (int64_t)gridDim.x * blockDim.x) {
        int col = 0;
        for (int c = 0; c < F.nkeys; c++, col++) {
            const FinalCol &o = F.out[col];
            bool n = F.gnull[c][g] != 0;
            o.nulls[g] = n ? 1 : 0;
            int64_t v = n ? 0 : F.gkey[c][g];
            if (o.type == GSQL_T_INT32) reinterpret_cast<int32_t *>(o.data)[g] = (int32_t)v;
            else reinterpret_cast<int64_t *>(o.data)[g] = v;  // INT64, or FP64 bits
        }
        for (int a = 0; a < F.naggs; a++, col++) {
            const FinalCol &o = F.out[col];
            const AggDev &ag = F.agg[a];
            long long lo, hi;
            o.nulls[g] = state_result(ag.kind, ag.in_type, state_load(ag, g), lo, hi) ? 1 : 0;
            if (o.type == GSQL_T_INT32) reinterpret_cast<int32_t *>(o.data)[g] = (int32_t)lo;
            else if (o.type == GSQL_T_DEC128) {
                reinterpret_cast<int64_t *>(o.data)[2 * g] = lo;
                reinterpret_cast<int64_t *>(o.data)[2 * g + 1] = hi;
            } else reinterpret_cast<int64_t *>(o.data)[g] = lo;  // INT64, or FP64 bits
        }
    }
}

int agg_out_type(int kind, int in_type) {
    switch (kind) {
    case GSQL_AGG_COUNT_STAR: case GSQL_AGG_COUNT: case GSQL_AGG_SUM0: return GSQL_T_INT64;
    case GSQL_AGG_SUM: return in_type == GSQL_T_FP64 ? GSQL_T_FP64 : GSQL_T_DEC128;
    case GSQL_AGG_AVG: case GSQL_AGG_AVG_MERGE: return GSQL_T_FP64;
    default: return in_type;  // MIN, MAX, FIRST_VALUE
    }
}

}  // namespace

// The rows a privatised front end (agg_smem, agg_lane, agg_reg) took, and how many of them missed its small tables and
// took the generic path.
struct FallbackRate {
    int64_t rows_seen = 0, rows_fallback = 0;
};

// Adds one launch to `r`; false once 2^16 rows or more have been seen and over 1/8 of them fell back: the key set does
// not fit the front end's tables, and it stops being chosen.
static bool still_profitable(FallbackRate &r, int64_t rows, int64_t fell) {
    r.rows_seen += rows;
    r.rows_fallback += fell;
    return !(r.rows_seen >= (1 << 16) && r.rows_fallback * 8 > r.rows_seen);
}

// Whether a privatised front end may take a batch: `shape_ok` is decided at create (the spec's aggregate kinds and key
// types), `enabled` adaptively (still_profitable, the group count).
struct AggFront {
    bool shape_ok = false, enabled = false;
    FallbackRate rate;
    bool usable() const { return shape_ok && enabled; }
    void disable() { shape_ok = enabled = false; }
};

#include "agg_fast.cuh"
#include "agg_lane.cuh"
#include "agg_reg.cuh"

struct gsql_agg {
    gsql_ctx *ctx;
    gsql_agg_spec spec;
    int32_t nkeys = 0, naggs = 0;
    int32_t in_type[GSQL_MAX_AGGS];
    int32_t nout = 0;
    int32_t out_types[GSQL_MAX_COLS];
    // table + state
    DevBuf slots, counters, overflow;
    uint64_t nslots = 0;
    int64_t gcap = 0, garr = 0;  // grow threshold, array capacity (gcap + slack)
    int64_t slack = 0;
    DevBuf gkey[GSQL_MAX_KEYS], gnull[GSQL_MAX_KEYS];
    DevBuf sl[GSQL_MAX_AGGS], shi[GSQL_MAX_AGGS], sd[GSQL_MAX_AGGS], shas[GSQL_MAX_AGGS];
    int64_t ngroups = 0;
    bool finished = false;
    DevBuf out_data[GSQL_MAX_COLS], out_nulls[GSQL_MAX_COLS];
    int64_t cursor = 0;
    AggFront reg, lane, smem;  // the privatised front ends (agg_launch)
    SmemLayout smem_layout;    // k_agg_smem's warp tables
    // tuning switches (INTEGRATION §7), read at create
    int part_on = 1;
    int64_t part_min_rows = 1ll << 22, part_bytes = 16ll << 20;
    int reg_stages = RGP_MAX_STAGES;  // k_agg_reg_pipe runs the stages that fit, at most reg_stages and at least 3
    int64_t fallback_total = 0;  // counters[C_FALLBACK] as of the last read (cumulative on the device)
    bool has_first_value = false;
    int64_t consumes = 0;        // consume calls with rows so far: FIRST_VALUE's ordinal
};

// (Re)allocates slots and state arrays for `gcap` groups, keeping the first `keep` groups' keys and states.
static gsql_status agg_resize(gsql_agg *a, int64_t gcap, int64_t keep) {
    gsql_ctx *ctx = a->ctx;
    int64_t garr = gcap + a->slack;
    uint64_t nslots = (uint64_t)(2 * garr);
    DevBuf nslot;
    GSQL_TRY(nslot.alloc(ctx, (size_t)(nslots + 2) * sizeof(ASlot)));
    {
        KernelScope ks(ctx, "agg_slots_init");
        k_aslots_init<<<grid_for(ctx, (int64_t)nslots + 2, 256, 8), 256, 0, ctx->stream>>>(nslot.as<ASlot>(), nslots + 2);
    }
    a->slots.release();
    a->slots.ctx = ctx;
    a->slots.p = nslot.p;
    a->slots.bytes = nslot.bytes;
    nslot.p = nullptr;
    a->nslots = nslots;
    for (int k = 0; k < a->nkeys; k++) {
        GSQL_TRY(a->gkey[k].grow(ctx, (size_t)garr * 8, (size_t)keep * 8));
        GSQL_TRY(a->gnull[k].grow(ctx, (size_t)garr, (size_t)keep));
    }
    for (int i = 0; i < a->naggs; i++) {
        const int kind = a->spec.aggs[i].kind;
        const AggStateArrays A = agg_state_arrays(kind, a->in_type[i]);
        const int64_t w = A.l_words;
        GSQL_TRY(a->sl[i].grow(ctx, (size_t)garr * 8 * w, (size_t)keep * 8 * w));
        {
            KernelScope ks(ctx, "agg_state_init");
            k_fill_i64<<<grid_for(ctx, (garr - keep) * w, 256, 8), 256, 0, ctx->stream>>>(a->sl[i].as<int64_t>(), A.l_init, keep * w, garr * w);
        }
        if (kind == GSQL_AGG_FIRST_VALUE && a->shi[i].p == nullptr) {  // the one-group cell, FV_EMPTY
            GSQL_TRY(a->shi[i].alloc(ctx, sizeof(FvCell)));
            GSQL_CUDA(ctx, cudaMemsetAsync(a->shi[i].p, 0xff, sizeof(FvCell), ctx->stream));
        }
        GSQL_TRY(a->shas[i].grow(ctx, (size_t)garr, (size_t)keep));
        GSQL_CUDA(ctx, cudaMemsetAsync((char *)a->shas[i].p + keep, 0, (size_t)(garr - keep), ctx->stream));
        if (A.hi) {
            GSQL_TRY(a->shi[i].grow(ctx, (size_t)garr * 8, (size_t)keep * 8));
            GSQL_CUDA(ctx, cudaMemsetAsync((char *)a->shi[i].p + keep * 8, 0, (size_t)(garr - keep) * 8, ctx->stream));
        }
        if (A.d) {
            GSQL_TRY(a->sd[i].grow(ctx, (size_t)garr * 8, (size_t)keep * 8));
            GSQL_CUDA(ctx, cudaMemsetAsync((char *)a->sd[i].p + keep * 8, 0, (size_t)(garr - keep) * 8, ctx->stream));
        }
    }
    a->gcap = gcap;
    a->garr = garr;
    return GSQL_OK;
}

static void agg_fill_params(gsql_agg *a, const StagedBatch *sb, AggParams *P) {
    memset(P, 0, sizeof(*P));
    if (sb) {
        P->in.n = sb->ncols;
        for (int i = 0; i < sb->ncols; i++) P->in.c[i] = sb->cols[i];
        P->keys.n = a->nkeys;
        for (int k = 0; k < a->nkeys; k++) {
            P->keys.c[k] = sb->cols[a->spec.groups[k]];
            P->keys.utype[k] = a->spec.input_types[a->spec.groups[k]];
        }
    }
    P->nkeys = a->nkeys;
    P->naggs = a->naggs;
    P->exact = a->nkeys == 1;
    P->slots = a->slots.as<ASlot>();
    P->nslots = a->nslots;
    for (int k = 0; k < a->nkeys; k++) {
        P->gkey[k] = a->gkey[k].as<int64_t>();
        P->gnull[k] = a->gnull[k].as<uint8_t>();
    }
    for (int i = 0; i < a->naggs; i++)
        P->agg[i] = agg_dev(a->spec.aggs[i], a->in_type[i], a->sl[i].as<int64_t>(), a->shi[i].as<int64_t>(), a->sd[i].as<double>(),
                            a->shas[i].as<uint8_t>());
    P->counters = a->counters.as<unsigned long long>();
    P->overflow_rows = a->overflow.as<int64_t>();
    P->gcap = a->gcap;
    P->garr = a->garr;
    for (int k = 0; k < a->nkeys; k++) P->keycol[k] = a->spec.groups[k];
    P->n_derived = a->spec.n_derived;
    for (int i = 0; i < a->spec.n_derived; i++) P->derived[i] = a->spec.derived[i];
    P->rf_col = a->spec.row_filter_col;
    P->rf_op = a->spec.row_filter_op;
    P->rf_value = a->spec.row_filter_value;
}

// Checks a gsql_agg_spec (shared by the hash and the sorted aggregation) and derives each aggregate's input type and the
// output schema (group keys, then one column per aggregate).
static gsql_status agg_check_spec(gsql_ctx *ctx, const gsql_agg_spec &s, int32_t *in_type, int32_t *out_types, int32_t *nout) {
    if (s.n_input_cols < 0 || s.n_input_cols > GSQL_MAX_COLS || s.ngroups < 0 || s.ngroups > GSQL_MAX_KEYS || s.naggs < 0 || s.naggs > GSQL_MAX_AGGS)
        return gsql_set_error(ctx, GSQL_E_INVALID, "bad agg spec sizes");
    if (s.ngroups + s.naggs > GSQL_MAX_COLS) return gsql_set_error(ctx, GSQL_E_INVALID, "too many output columns");
    for (int i = 0; i < s.n_input_cols; i++)
        if (s.input_types[i] < GSQL_T_INT32 || s.input_types[i] > GSQL_T_FP64) return gsql_set_error(ctx, GSQL_E_UNSUPPORTED, "input col %d type", i);
    for (int k = 0; k < s.ngroups; k++)
        if (s.groups[k] < 0 || s.groups[k] >= s.n_input_cols) return gsql_set_error(ctx, GSQL_E_INVALID, "group col out of range");
    if (s.n_derived < 0 || s.n_derived > GSQL_MAX_DERIVED) return gsql_set_error(ctx, GSQL_E_INVALID, "bad derived column count");
    for (int i = 0; i < s.n_derived; i++) {
        const gsql_derived_col &d = s.derived[i];
        if (d.kind != GSQL_EXPR_MUL_1MINUS && d.kind != GSQL_EXPR_MUL_1MINUS_1PLUS) return gsql_set_error(ctx, GSQL_E_UNSUPPORTED, "derived column %d: expression kind", i);
        int nops = d.kind == GSQL_EXPR_MUL_1MINUS ? 2 : 3;
        const int ops[3] = {d.a, d.b, d.c};
        for (int q = 0; q < nops; q++)
            if (ops[q] < 0 || ops[q] >= s.n_input_cols) return gsql_set_error(ctx, GSQL_E_INVALID, "derived column %d: operand out of range", i);
    }
    if (s.row_filter_op != GSQL_CMP_NONE) {
        if (s.row_filter_op < GSQL_CMP_LE || s.row_filter_op > GSQL_CMP_NE || s.row_filter_col < 0 || s.row_filter_col >= s.n_input_cols ||
            s.input_types[s.row_filter_col] == GSQL_T_FP64)
            return gsql_set_error(ctx, GSQL_E_UNSUPPORTED, "row filter must compare an INT/BIGINT input column");
    }
    *nout = 0;
    for (int k = 0; k < s.ngroups; k++) out_types[(*nout)++] = s.input_types[s.groups[k]];
    for (int i = 0; i < s.naggs; i++) {
        const gsql_agg_call &c = s.aggs[i];
        if (c.kind < GSQL_AGG_COUNT_STAR || c.kind > GSQL_AGG_FIRST_VALUE) return gsql_set_error(ctx, GSQL_E_UNSUPPORTED, "agg kind %d", c.kind);
        int need = c.kind == GSQL_AGG_COUNT_STAR ? 0 : 1;
        if (c.kind == GSQL_AGG_AVG_MERGE) need = 2;
        if (c.ncols < need || c.ncols > 4 || (c.kind != GSQL_AGG_COUNT && c.kind != GSQL_AGG_COUNT_STAR && c.ncols != need)) return gsql_set_error(ctx, GSQL_E_INVALID, "agg %d: argument count", i);
        for (int q = 0; q < c.ncols; q++)
            if (c.cols[q] < 0 || c.cols[q] >= s.n_input_cols + s.n_derived) return gsql_set_error(ctx, GSQL_E_INVALID, "agg %d: column out of range", i);
        if (c.filter_arg >= s.n_input_cols) return gsql_set_error(ctx, GSQL_E_INVALID, "agg %d: filter column", i);
        in_type[i] = c.ncols > 0 ? (c.cols[0] < s.n_input_cols ? s.input_types[c.cols[0]] : GSQL_T_FP64) : GSQL_T_INT64;
        // planner-time fall-through cases (the stock HashAggExec keeps them): AVG over integers is DECIMAL division
        if (c.kind == GSQL_AGG_AVG && in_type[i] != GSQL_T_FP64) return gsql_set_error(ctx, GSQL_E_UNSUPPORTED, "AVG(integer) -> DECIMAL not on the GPU path");
        if (c.kind == GSQL_AGG_AVG_MERGE && (in_type[i] != GSQL_T_FP64 || c.cols[1] >= s.n_input_cols || s.input_types[c.cols[1]] != GSQL_T_INT64)) return gsql_set_error(ctx, GSQL_E_UNSUPPORTED, "AVG_MERGE needs (DOUBLE partial sum, BIGINT partial count)");
        if (c.kind == GSQL_AGG_SUM0 && in_type[i] != GSQL_T_INT64) return gsql_set_error(ctx, GSQL_E_UNSUPPORTED, "SUM0 needs BIGINT input");
        // InternalFirstValue with a FILTER argument: a group whose first row is filtered out leaves the stock aggregator's
        // value buffer one entry short, and the next new group fails.  Refused rather than restated differently.
        if (c.kind == GSQL_AGG_FIRST_VALUE && c.filter_arg >= 0) return gsql_set_error(ctx, GSQL_E_UNSUPPORTED, "agg %d: FIRST_VALUE with a FILTER argument", i);
        out_types[(*nout)++] = agg_out_type(c.kind, in_type[i]);
    }
    return GSQL_OK;
}

extern "C" gsql_status gsql_agg_create(gsql_ctx *ctx, const gsql_agg_spec *spec, gsql_agg **out) {
    if (!ctx || !spec || !out) return GSQL_E_INVALID;
    if (ctx->sticky) return GSQL_E_CUDA;
    *out = nullptr;
    const gsql_agg_spec &s = *spec;
    int32_t in_type[GSQL_MAX_AGGS], out_types[GSQL_MAX_COLS], nout = 0;
    GSQL_TRY(agg_check_spec(ctx, s, in_type, out_types, &nout));
    gsql_agg *a = new gsql_agg();
    a->ctx = ctx;
    gsql_ctx_retain(ctx);
    a->spec = s;
    a->nkeys = s.ngroups;
    a->naggs = s.naggs;
    a->nout = nout;
    memcpy(a->in_type, in_type, sizeof(in_type));
    memcpy(a->out_types, out_types, sizeof(out_types));
    cudaSetDevice(ctx->device);
    agg_reg_check(&a->reg, a->spec, a->nkeys, a->naggs, a->spec.aggs, a->in_type);
    agg_lane_check(&a->lane, a->spec, a->nkeys, a->naggs, a->spec.aggs, a->in_type);
    agg_fast_plan(&a->smem, &a->smem_layout, a->spec, a->nkeys, a->naggs, a->spec.aggs, a->in_type);
    if (s.expected_groups > (1 << 16)) a->smem.enabled = false;  // the planner expects far more groups than warp tables hold
    for (int i = 0; i < s.naggs; i++)
        if (s.aggs[i].kind == GSQL_AGG_AVG_MERGE || s.aggs[i].kind == GSQL_AGG_FIRST_VALUE) {
            // the privatised kernels know neither the two-column merge nor the row order FIRST_VALUE needs
            a->has_first_value |= s.aggs[i].kind == GSQL_AGG_FIRST_VALUE;
            a->reg.disable();
            a->lane.disable();
            a->smem.disable();
        }
    int no_reg = 0, no_lane = 0, no_fast = 0;
    if (env_knob("GSQL_AGG_NO_REG", &no_reg) && no_reg) a->reg.disable();
    if (env_knob("GSQL_AGG_NO_LANE", &no_lane) && no_lane) a->lane.disable();
    if (env_knob("GSQL_AGG_NO_FAST", &no_fast) && no_fast) { a->lane.disable(); a->smem.disable(); }
    env_knob("GSQL_AGG_PARTITION", &a->part_on);
    env_knob("GSQL_AGG_PARTITION_MIN_ROWS", &a->part_min_rows);
    env_knob("GSQL_AGG_PARTITION_BYTES", &a->part_bytes);
    // any value, 0 included, caps the pipeline depth (at least 3); unset, the cap RGP_MAX_STAGES changes nothing
    env_knob("GSQL_AGG_REG_STAGES", &a->reg_stages);
    a->slack = (int64_t)ctx->sm_count * 2048 + 1024 + (int64_t)ctx->sm_count * 2 * 1024;  // + CTA-table merges of the smem path
    int64_t gcap = s.expected_groups > 0 ? s.expected_groups : 1024;
    if (gcap < 65536) gcap = 65536;
    gsql_status st = a->counters.alloc(ctx, C_COUNT * 8);
    if (st == GSQL_OK) st = (cudaMemsetAsync(a->counters.p, 0, C_COUNT * 8, ctx->stream) == cudaSuccess) ? GSQL_OK : GSQL_E_CUDA;
    if (st == GSQL_OK) st = agg_resize(a, gcap, 0);
    if (st == GSQL_OK && a->nkeys == 0) {  // noGroupBy: one group exists from the start (AggOpenHashMap.java:93-96)
        unsigned long long one = 1;
        cudaMemcpyAsync(a->counters.p, &one, 8, cudaMemcpyHostToDevice, ctx->stream);
        cudaStreamSynchronize(ctx->stream);
        a->ngroups = 1;
    }
    if (st != GSQL_OK) { delete a; gsql_ctx_release(ctx); return st; }
    *out = a;
    return GSQL_OK;
}

extern "C" void gsql_agg_destroy(gsql_agg *a) { destroy_handle(a); }

static gsql_status agg_read_counters(gsql_agg *a, unsigned long long *h) {
    gsql_ctx *ctx = a->ctx;
    GSQL_CUDA(ctx, cudaMemcpyAsync(h, a->counters.p, C_COUNT * 8, cudaMemcpyDeviceToHost, ctx->stream));
    GSQL_CUDA(ctx, cudaStreamSynchronize(ctx->stream));
    return GSQL_OK;
}

// Calls f(NK) with NK = nkeys for 1..3 group keys and NK = 0 (the dynamic form) otherwise, NK as a compile-time
// constant for the kernel's template argument: that keeps the key image in registers (see digest_of_keys).
template <typename F>
static auto with_nkeys(int nkeys, F &&f) {
    switch (nkeys) {
    case 1: return f(std::integral_constant<int, 1>{});
    case 2: return f(std::integral_constant<int, 2>{});
    case 3: return f(std::integral_constant<int, 3>{});
    default: return f(std::integral_constant<int, 0>{});
    }
}

// Calls f(NS, G) with the register kernels' instantiation for `nsrc` distinct fp64 sums: NS = nsrc (at most RG_MAX_SRC),
// G = the groups a block holds in registers, 8 up to four sums and 6 beyond (RG_G).
template <typename F>
static auto with_reg_shape(int nsrc, F &&f) {
    switch (nsrc) {
    case 1: return f(std::integral_constant<int, 1>{}, std::integral_constant<int, 8>{});
    case 2: return f(std::integral_constant<int, 2>{}, std::integral_constant<int, 8>{});
    case 3: return f(std::integral_constant<int, 3>{}, std::integral_constant<int, 8>{});
    case 4: return f(std::integral_constant<int, 4>{}, std::integral_constant<int, 8>{});
    case 5: return f(std::integral_constant<int, 5>{}, std::integral_constant<int, 6>{});
    default: return f(std::integral_constant<int, 6>{}, std::integral_constant<int, 6>{});
    }
}

// Reorders the staged batch by table-slot range (see k_agg_part_hist).  `sb` is rewritten to point at the reordered
// columns, which live in `bufs` until the caller returns.
static gsql_status agg_partition_batch(gsql_agg *a, StagedBatch *sb, int nparts, DevBuf *bufs, DevBuf *nbufs) {
    gsql_ctx *ctx = a->ctx;
    {  // the C5 shape — one integer key, a few NULL-free columns — goes through the warp-synchronous split kernels of the
       // push exchange (xchg.cu); the scalar scatter below is latency-bound
        bool plain = a->nkeys == 1 && sb->ncols <= 4 && nparts <= GSQL_MAX_RANKS && sb->cols[a->spec.groups[0]].type != GSQL_T_FP64;
        for (int c = 0; c < sb->ncols; c++) plain = plain && sb->cols[c].nulls == nullptr;
        if (plain) {
            DColSet in;
            memset(&in, 0, sizeof(in));
            in.n = sb->ncols;
            void *out[GSQL_MAX_COLS];
            for (int c = 0; c < sb->ncols; c++) {
                in.c[c] = sb->cols[c];
                GSQL_TRY(bufs[c].alloc(ctx, (size_t)sb->rows * gsql_type_width(sb->cols[c].type)));
                out[c] = bufs[c].p;
            }
            GSQL_TRY(local_split_by_slot_range(ctx, in, a->spec.groups[0], sb->rows, nparts, out));
            for (int c = 0; c < sb->ncols; c++) sb->cols[c].data = out[c];
            return GSQL_OK;
        }
    }
    AggParams P;
    agg_fill_params(a, sb, &P);
    P.row0 = 0;
    P.rows = sb->rows;
    APart G;
    int nblocks = grid_for(ctx, sb->rows, 4096, 8);
    G.chunk = div_up(div_up(sb->rows, nblocks), 256) * 256;
    nblocks = (int)div_up(sb->rows, G.chunk);
    if (nblocks < 1) nblocks = 1;
    G.nblocks = nblocks;
    G.nparts = nparts;
    int64_t nh = (int64_t)nparts * nblocks;
    DevBuf hist, offs, tmp;
    GSQL_TRY(hist.alloc(ctx, (size_t)(nh + 1) * 8));
    GSQL_TRY(offs.alloc(ctx, (size_t)(nh + 1) * 8));
    GSQL_CUDA(ctx, cudaMemsetAsync((char *)hist.p + nh * 8, 0, 8, ctx->stream));
    {
        KernelScope ks(ctx, "agg_part_hist");
        with_nkeys(a->nkeys, [&](auto nk) {
            k_agg_part_hist<nk><<<nblocks, 256, (size_t)nparts * sizeof(unsigned int), ctx->stream>>>(P, G, hist.as<int64_t>());
        });
    }
    GSQL_CUDA(ctx, cudaGetLastError());
    size_t tb = 0;
    GSQL_CUDA(ctx, cub::DeviceScan::ExclusiveSum(nullptr, tb, hist.as<int64_t>(), offs.as<int64_t>(), nh + 1, ctx->stream));
    GSQL_TRY(tmp.alloc(ctx, tb));
    GSQL_CUDA(ctx, cub::DeviceScan::ExclusiveSum(tmp.p, tb, hist.as<int64_t>(), offs.as<int64_t>(), nh + 1, ctx->stream));
    APartOut O;
    memset(&O, 0, sizeof(O));
    for (int c = 0; c < sb->ncols; c++) {
        GSQL_TRY(bufs[c].alloc(ctx, (size_t)sb->rows * gsql_type_width(sb->cols[c].type)));
        O.data[c] = bufs[c].p;
        if (sb->cols[c].nulls) {
            GSQL_TRY(nbufs[c].alloc(ctx, (size_t)sb->rows));
            O.nulls[c] = nbufs[c].as<uint8_t>();
        }
    }
    {
        KernelScope ks(ctx, "agg_part_scatter");
        with_nkeys(a->nkeys, [&](auto nk) {
            k_agg_part_scatter<nk><<<nblocks, 256, (size_t)nparts * sizeof(unsigned long long), ctx->stream>>>(P, G, offs.as<int64_t>(), O);
        });
    }
    GSQL_CUDA(ctx, cudaGetLastError());
    for (int c = 0; c < sb->ncols; c++) {
        sb->cols[c].data = O.data[c];
        sb->cols[c].nulls = O.nulls[c];
    }
    return GSQL_OK;
}

// Launches register kernel `name`<ns, g> with `smem` bytes of dynamic shared memory.  A failure to raise the kernel's limit
// is reported as GSQL_CUDA reports it, with the instantiation's template arguments spelled out.
template <typename K>
static gsql_status reg_launch(gsql_ctx *ctx, K *kernel, const char *name, int ns, int g, int grid, int threads, size_t smem,
                              const AggParams &P, const RegPlan &L) {
    const cudaError_t e = cudaFuncSetAttribute(kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem);
    if (e != cudaSuccess) {
        ctx->sticky = true;
        return gsql_set_error(ctx, e == cudaErrorMemoryAllocation ? GSQL_E_OOM : GSQL_E_CUDA,
                              "%s:%d cudaFuncSetAttribute(%s<%d, %d>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem) -> %s", __FILE__,
                              __LINE__, name, ns, g, cudaGetErrorString(e));
    }
    kernel<<<grid, threads, smem, ctx->stream>>>(P, L);
    return GSQL_OK;
}

// The slot-range pre-pass: a large batch headed for the generic kernel against a table beyond L2 is first reordered by
// table-slot range (GSQL_AGG_PARTITION=0 switches it off).  "Headed for the generic kernel" is judged from the front
// ends' create-time and adaptive state alone, not from this batch's plans (agg_launch).  The reordered columns live in
// `part_data` / `part_nulls` until the caller returns.
static gsql_status agg_prepass(gsql_agg *a, StagedBatch *sb, DevBuf *part_data, DevBuf *part_nulls) {
    const bool generic = !a->reg.usable() && !a->lane.usable() && !a->smem.usable();
    const int64_t per_group = 2 * (int64_t)sizeof(ASlot) + (int64_t)a->nkeys * 9 + (int64_t)a->naggs * 9;
    const int64_t table_bytes = (a->gcap + a->slack) * per_group;
    const int64_t slice = a->part_bytes;
    // Not with FIRST_VALUE: its row tags need the positions as passed, and on the TPC-H Q18 shape (225 M rows, 56 M groups,
    // H100 80GB HBM3 at 700 W) the spec ran faster without the pre-pass than with it carrying them (tools/firstvaluebench.py,
    // DESIGN §4)
    if (!a->part_on || !generic || a->has_first_value || a->nkeys == 0 || sb->rows < a->part_min_rows || table_bytes <= 4 * slice)
        return GSQL_OK;
    int64_t nparts = div_up(table_bytes, slice);
    // up to 16 partitions the fast split kernels apply: prefer somewhat larger slices (<= 32 MB) to the scalar scatter
    if (nparts > GSQL_MAX_RANKS && div_up(table_bytes, GSQL_MAX_RANKS) <= 2 * slice) nparts = GSQL_MAX_RANKS;
    if (nparts > 4096) nparts = 4096;
    return agg_partition_batch(a, sb, (int)nparts, part_data, part_nulls);
}

// Launches one pass over P's rows on the most specialised front end that takes them: register accumulators (NULL-free
// batch, <= 8 groups, fp64 sums: the Q1 shape), lane-private accumulators (a handful of groups), warp-private
// shared-memory tables (tens of groups), else the generic global table.  The privatised three are adaptive and are
// tried on a batch's first pass only; overflow re-runs take the generic kernel.  *ran: the front end that ran, nullptr
// for the generic kernel.
static gsql_status agg_launch(gsql_agg *a, const AggParams &P, bool first, AggFront **ran) {
    gsql_ctx *ctx = a->ctx;
    RegPlan RP;
    LanePlan LP;
    AggFront *f = nullptr;
    if (first && a->reg.usable() && agg_reg_plan(&RP, a->spec, a->nkeys, a->naggs, a->spec.aggs, P.in)) f = &a->reg;
    else if (first && a->lane.usable() && agg_lane_plan(&LP, a->spec, a->nkeys, a->naggs, a->spec.aggs, a->in_type, P.in)) f = &a->lane;
    else if (first && a->smem.usable()) f = &a->smem;
    *ran = f;
    if (f == &a->reg) {
        KernelScope ks(ctx, "agg_reg");
        // bulk-copy staging needs 16-byte aligned sources; tiles start at multiples of 512 rows, so only the base counts
        bool aligned = true;
        for (int u = 0; u < RP.nused; u++) {
            const DCol &c = P.in.c[RP.used_col[u]];
            if ((reinterpret_cast<uintptr_t>(c.data) + (uintptr_t)P.row0 * (uintptr_t)RP.used_w[u]) % 16 != 0) aligned = false;
        }
        if (aligned) {  // k_agg_reg_pipe: 512-row tiles, 3-4 stages, full / empty mbarriers
            RegPlan PP;
            agg_reg_plan(&PP, a->spec, a->nkeys, a->naggs, a->spec.aggs, P.in, RGP_TILE);  // same verdict as RP, other tile size
            // two blocks per SM, 104 KB of tile buffers each: even the largest tile (RG_MAX_USED 8-byte columns, 32 KB)
            // fits 3 stages
            constexpr size_t budget2 = (size_t)104 * 1024;
            static_assert(budget2 / ((size_t)RGP_TILE * RG_MAX_USED * 8) >= 3, "the largest pipe tile must fit 3 stages");
            PP.stages = std::max(3, std::min((int)std::min<size_t>(RGP_MAX_STAGES, budget2 / PP.tile_bytes), a->reg_stages));
            const size_t smem = (size_t)PP.stages * PP.tile_bytes;
            const int grid = grid_for(ctx, P.rows, RGP_TILE, 2);
            return with_reg_shape(PP.nsrc, [&](auto ns, auto g) { return reg_launch(ctx, k_agg_reg_pipe<ns, g>, "k_agg_reg_pipe", ns, g, grid, RGP_THREADS, smem, P, PP); });
        }
        // k_agg_reg: 1024-row tiles, two buffers, per-thread cp.async
        const size_t smem = (size_t)2 * RP.tile_bytes;
        const int grid = grid_for(ctx, P.rows, RG_TILE, smem * 2 + 16384 <= 220 * 1024 ? 2 : 1);
        return with_reg_shape(RP.nsrc, [&](auto ns, auto g) { return reg_launch(ctx, k_agg_reg<ns, g>, "k_agg_reg", ns, g, grid, RG_THREADS, smem, P, RP); });
    }
    if (f == &a->lane) {
        KernelScope ks(ctx, "agg_lane");
        const int grid = grid_for(ctx, P.rows, 32 * LA_R * LA_WARPS, 1);
        // per device, cheap: set before every launch (a process may drive several GPUs through several contexts)
        GSQL_CUDA(ctx, cudaFuncSetAttribute(k_agg_lane, cudaFuncAttributeMaxDynamicSharedMemorySize, LP.total));
        k_agg_lane<<<grid, LA_THREADS, LP.total, ctx->stream>>>(P, LP);
        return GSQL_OK;
    }
    if (f == &a->smem) {
        KernelScope ks(ctx, "agg_smem");
        const int grid = grid_for(ctx, P.rows, AF_THREADS, 2);
        GSQL_CUDA(ctx, cudaFuncSetAttribute(k_agg_smem, cudaFuncAttributeMaxDynamicSharedMemorySize, a->smem_layout.total));
        k_agg_smem<<<grid, AF_THREADS, a->smem_layout.total, ctx->stream>>>(P, a->smem_layout);
        return GSQL_OK;
    }
    KernelScope ks(ctx, "agg_consume");
    const int grid = grid_for(ctx, P.rows, 256, 8);
    with_nkeys(a->nkeys, [&](auto nk) {
        if (a->has_first_value) k_agg_consume_fv<nk><<<grid, 256, 0, ctx->stream>>>(P);
        else k_agg_consume<nk><<<grid, 256, 0, ctx->stream>>>(P);
    });
    return GSQL_OK;
}

extern "C" gsql_status gsql_agg_consume(gsql_agg *a, const gsql_batch *batch) {
    if (!a) return GSQL_E_INVALID;
    gsql_ctx *ctx = a->ctx;
    if (ctx->sticky) return GSQL_E_CUDA;
    if (a->finished) return gsql_set_error(ctx, GSQL_E_STATE, "consume after finish");
    GSQL_TRY(validate_batch(ctx, batch, a->spec.n_input_cols, a->spec.input_types));
    if (batch->rows == 0) return GSQL_OK;
    GSQL_CUDA(ctx, cudaSetDevice(ctx->device));
    gsql_batch stripped;
    gsql_col stripped_cols[GSQL_MAX_COLS];
    {  // all-zero null masks are dropped: the privatised kernels keep their no-NULL shortcuts for a caller that always passes isNull[]
        bool has_mask = false;
        for (int i = 0; i < batch->ncols; i++) has_mask |= batch->cols[i].nulls != nullptr;
        if (has_mask) {
            GSQL_TRY(strip_zero_masks(ctx, batch, &stripped, stripped_cols));
            batch = &stripped;
        }
    }
    StagedBatch sb;
    GSQL_TRY(stage_batch(ctx, batch, &sb));
    GSQL_TRY(a->overflow.grow(ctx, (size_t)batch->rows * 8, 0));
    if (a->has_first_value) {  // the row tag's fields (GSQL_AGG_FIRST_VALUE) must not wrap
        if (a->consumes >= FV_MAX_ORDINAL) return gsql_set_error(ctx, GSQL_E_CAPACITY, "FIRST_VALUE: more than %lld consume calls", (long long)FV_MAX_ORDINAL);
        if (batch->rows >= (1LL << FV_POS_BITS)) return gsql_set_error(ctx, GSQL_E_CAPACITY, "FIRST_VALUE: a batch of %lld rows is too large", (long long)batch->rows);
    }
    DevBuf part_data[GSQL_MAX_COLS], part_nulls[GSQL_MAX_COLS];
    GSQL_TRY(agg_prepass(a, &sb, part_data, part_nulls));
    AggParams P;
    agg_fill_params(a, &sb, &P);
    P.row0 = 0;
    P.rows = batch->rows;
    P.row_list = nullptr;
    const unsigned long long fv_tag0 = (unsigned long long)a->consumes++ << FV_ORD_SHIFT;
    P.fv_tag0 = fv_tag0;
    DevBuf pending;  // overflow rows being re-run
    for (bool first = true;; first = false) {
        AggFront *ran;
        GSQL_TRY(agg_launch(a, P, first, &ran));
        GSQL_CUDA(ctx, cudaGetLastError());
        unsigned long long h[C_COUNT];
        GSQL_TRY(agg_read_counters(a, h));
        {  // adaptive: stop using a privatised kernel when its small tables do not hold the key set
            const int64_t fell = (int64_t)h[C_FALLBACK] - a->fallback_total;
            a->fallback_total = (int64_t)h[C_FALLBACK];
            if (ran) ran->enabled = still_profitable(ran->rate, P.rows, fell);
        }
        a->ngroups = (int64_t)h[C_NGROUPS];
        if (h[C_FATAL]) {
            ctx->sticky = true;
            return gsql_set_error(ctx, GSQL_E_CAPACITY, "group arrays overflowed (%lld groups, capacity %lld)", (long long)a->ngroups, (long long)a->garr);
        }
        // the privatised kernels merge warp-private groups past gcap (into the slack): beyond a few tens of thousands of
        // groups they cannot win any more, and every launch may add warps x S groups unchecked
        if (a->ngroups > (1 << 16)) a->reg.enabled = a->lane.enabled = a->smem.enabled = false;
        int64_t nover = (int64_t)h[C_OVERFLOW];
        if (nover == 0) {
            // merges that ignored the cap may have eaten into the slack: restore it before the next launch
            if (a->ngroups > a->gcap) {
                int64_t ncap = a->gcap * 2;
                while (ncap < a->ngroups) ncap *= 2;
                GSQL_TRY(agg_resize(a, ncap, a->ngroups));
                agg_fill_params(a, &sb, &P);
                KernelScope ks(ctx, "agg_rehash");
                k_agg_rehash<<<grid_for(ctx, a->ngroups, 256, 8), 256, 0, ctx->stream>>>(P, a->ngroups);
                GSQL_CUDA(ctx, cudaGetLastError());
            }
            break;
        }
        // table full: double (at least) the group capacity, re-insert the groups, re-run only the overflowed rows
        GSQL_TRY(pending.alloc(ctx, (size_t)nover * 8));
        GSQL_CUDA(ctx, cudaMemcpyAsync(pending.p, a->overflow.p, (size_t)nover * 8, cudaMemcpyDeviceToDevice, ctx->stream));
        unsigned long long zero = 0;
        GSQL_CUDA(ctx, cudaMemcpyAsync(a->counters.as<unsigned long long>() + C_OVERFLOW, &zero, 8, cudaMemcpyHostToDevice, ctx->stream));
        int64_t ncap = a->gcap * 2;
        while (ncap < a->ngroups + nover / 4) ncap *= 2;
        GSQL_TRY(agg_resize(a, ncap, a->ngroups));
        agg_fill_params(a, &sb, &P);
        {
            KernelScope ks(ctx, "agg_rehash");
            k_agg_rehash<<<grid_for(ctx, a->ngroups, 256, 8), 256, 0, ctx->stream>>>(P, a->ngroups);
        }
        GSQL_CUDA(ctx, cudaGetLastError());
        P.row_list = pending.as<int64_t>();  // original row positions: FIRST_VALUE's tags stay those of the first pass
        P.rows = nover;
        P.fv_tag0 = fv_tag0;
    }
    if (batch->mem == GSQL_MEM_HOST) GSQL_CUDA(ctx, cudaStreamSynchronize(ctx->stream));
    return GSQL_OK;
}

extern "C" gsql_status gsql_agg_output_schema(gsql_agg *a, int32_t *ncols, int32_t *types) {
    if (!a || !ncols) return GSQL_E_INVALID;
    return output_schema(a->nout, a->out_types, ncols, types);
}

extern "C" gsql_status gsql_agg_finish(gsql_agg *a, int64_t *ngroups) {
    if (!a) return GSQL_E_INVALID;
    gsql_ctx *ctx = a->ctx;
    if (ctx->sticky) return GSQL_E_CUDA;
    GSQL_CUDA(ctx, cudaSetDevice(ctx->device));
    if (!a->finished) {
        int64_t n = a->ngroups;
        FinalParams F;
        memset(&F, 0, sizeof(F));
        F.nkeys = a->nkeys;
        F.naggs = a->naggs;
        F.ngroups = n;
        AggParams P;
        agg_fill_params(a, nullptr, &P);
        for (int k = 0; k < a->nkeys; k++) {
            F.gkey[k] = P.gkey[k];
            F.gnull[k] = P.gnull[k];
            F.key_types[k] = a->out_types[k];
        }
        for (int i = 0; i < a->naggs; i++) F.agg[i] = P.agg[i];
        for (int c = 0; c < a->nout; c++) {
            GSQL_TRY(a->out_data[c].alloc(ctx, (size_t)(n > 0 ? n : 1) * gsql_type_width(a->out_types[c])));
            GSQL_TRY(a->out_nulls[c].alloc(ctx, (size_t)(n > 0 ? n : 1)));
            F.out[c].data = a->out_data[c].p;
            F.out[c].nulls = a->out_nulls[c].as<uint8_t>();
            F.out[c].type = a->out_types[c];
        }
        if (n == 1)  // one group: FIRST_VALUE is its first non-NULL value instead (InternalFirstValue.writeResultTo:112-127)
            for (int i = 0; i < a->naggs; i++)
                if (a->spec.aggs[i].kind == GSQL_AGG_FIRST_VALUE)
                    GSQL_CUDA(ctx, cudaMemcpyAsync(a->sl[i].p, a->shi[i].p, sizeof(FvCell), cudaMemcpyDeviceToDevice, ctx->stream));
        if (n > 0) {
            KernelScope ks(ctx, "agg_finalize");
            k_agg_finalize<<<grid_for(ctx, n, 256, 8), 256, 0, ctx->stream>>>(F);
        }
        GSQL_CUDA(ctx, cudaGetLastError());
        a->finished = true;
        a->cursor = 0;
    }
    if (ngroups) *ngroups = a->ngroups;
    return GSQL_OK;
}

extern "C" gsql_status gsql_agg_next(gsql_agg *a, gsql_batch *out, int64_t max_rows, int64_t *out_rows) {
    if (!a || !out || !out_rows) return GSQL_E_INVALID;
    gsql_ctx *ctx = a->ctx;
    if (ctx->sticky) return GSQL_E_CUDA;
    if (!a->finished) return gsql_set_error(ctx, GSQL_E_STATE, "next before finish");
    GSQL_TRY(validate_batch(ctx, out, a->nout, a->out_types));
    GSQL_CUDA(ctx, cudaSetDevice(ctx->device));
    int64_t n = a->ngroups - a->cursor;
    if (n > max_rows) n = max_rows;
    if (n < 0) n = 0;
    *out_rows = n;
    out->rows = n;
    if (n == 0) return GSQL_OK;
    for (int c = 0; c < a->nout; c++) {
        if (!out->cols[c].nulls) return gsql_set_error(ctx, GSQL_E_INVALID, "agg output column %d needs a nulls buffer", c);
        GSQL_TRY(out_copy_rows(ctx, out, c, 0, a->out_data[c], a->out_nulls[c], a->cursor, n));
    }
    if (out->mem == GSQL_MEM_HOST) GSQL_CUDA(ctx, cudaStreamSynchronize(ctx->stream));
    a->cursor += n;
    return GSQL_OK;
}

#include "agg_sets.cuh"
#include "agg_sorted.cuh"
#include "window.cuh"
