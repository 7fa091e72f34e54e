// agg_state.cuh — what an aggregate's partial state is and what can be done with it, for every operator that aggregates:
// the hash aggregation and its front ends (agg.cu, agg_fast.cuh, agg_lane.cuh, agg_reg.cuh), grouping sets (agg_sets.cuh),
// the sorted aggregation (agg_sorted.cuh) and the window (window.cuh).  Included by agg.cu inside its anonymous namespace,
// after AggDev, FvCell and the sortable double image; the per-row folds stay with each operator.
//
// A group's state lives in the AggDev arrays, by group id:
//   l    COUNT / COUNT(*) / SUM0 | MIN / MAX (sortable image for DOUBLE) | SUM(int) low word | AVG row count |
//        FIRST_VALUE: one FvCell (two words) per group
//   hi   SUM(int) high word (only that kind has the array)
//   d    DOUBLE SUM / AVG sum (only those kinds have the array)
//   has  "the state is not NULL" (every kind has the array; the counts never set it)
// At rest a group whose has is 0 holds state_zero in its arrays (the operators fill l with it and zero hi and d, and every
// merge is gated on has), so state_load needs no NULL case: state_combine with it is the identity.
// In registers the state is an SState.  FIRST_VALUE's state is its cell's value and "a non-NULL value was seen": state_load reads
// the cell's NULL bit, state_store writes tag 0 (before every later part's tag) or FV_EMPTY.
#pragma once

struct SState {  // one aggregate's partial over a run of rows; also the segmented scans' element
    long long l;  // AggDev::l (FIRST_VALUE: the value bits, FvCell::val)
    long long x;  // AggDev::hi (SUM of integers) or the bits of AggDev::d (DOUBLE sums)
    int has;      // AggDev::has
    int f;        // scans only: a run starts in the rows this partial covers
};
__device__ __forceinline__ double sa_d(const SState &s) { return __longlong_as_double(s.x); }
__device__ __forceinline__ void sa_set_d(SState &s, double d) { s.x = __double_as_longlong(d); }

// The state of no rows: the identity of every combine and merge below (MIN / MAX: the sentinels atomicMin / atomicMax
// start from; sums +0.0).
__host__ __device__ __forceinline__ SState state_zero(int kind) {
    SState s{0, 0, 0, 0};
    if (kind == GSQL_AGG_MIN) s.l = 0x7fffffffffffffffLL;
    if (kind == GSQL_AGG_MAX) s.l = (long long)0x8000000000000000ULL;
    return s;
}

// a then b (b's rows follow a's).  FV = false: the caller never sees FIRST_VALUE.
template <bool FV = true>
__device__ __forceinline__ SState state_combine(int kind, int in_type, const SState &a, const SState &b) {
    SState s = a;
    s.has = a.has | b.has;
    if constexpr (FV) {
        if (kind == GSQL_AGG_FIRST_VALUE) {  // associative: the earlier part's value when it has one
            s.l = a.has ? a.l : b.l;
            return s;
        }
    }
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

// Group g's state, read from the arrays its kind uses.
__device__ __forceinline__ SState state_load(const AggDev &a, int64_t g) {
    SState s{0, 0, 0, 0};
    if (a.kind == GSQL_AGG_FIRST_VALUE) {
        const FvCell c = reinterpret_cast<const FvCell *>(a.l)[g];
        s.l = c.val;
        s.has = (c.tag & 1ULL) == 0;  // the NULL bit, set in FV_EMPTY too
        return s;
    }
    if (a.kind != GSQL_AGG_SUM || !a.d) s.l = a.l[g];  // a DOUBLE SUM keeps nothing in l
    if (a.hi) s.x = a.hi[g];
    if (a.d) s.x = __double_as_longlong(a.d[g]);
    s.has = a.has[g];
    return s;
}

// Stores s whole as group g's state.  FV = false: the caller never sees FIRST_VALUE.
template <bool FV = true>
__device__ __forceinline__ void state_store(const AggDev &a, int64_t g, const SState &s) {
    if (FV && a.kind == GSQL_AGG_FIRST_VALUE) {  // tag 0: before every part that follows (agg_sorted.cuh)
        reinterpret_cast<FvCell *>(a.l)[g] = FvCell{s.has ? 0ULL : FV_EMPTY, s.l};
        return;
    }
    a.l[g] = s.l;
    if (a.hi) a.hi[g] = s.x;
    if (a.d) a.d[g] = sa_d(s);
    a.has[g] = (uint8_t)s.has;
}

// Merges partial s into group gid with atomics, in any order with the other partials of the group.  A zero count and a
// NULL partial take no atomic.  FIRST_VALUE merges through fv_min, with the tag its caller knows the partial by.
__device__ __forceinline__ void state_merge(const AggDev &a, int64_t gid, const SState &s) {
    switch (a.kind) {
    case GSQL_AGG_COUNT_STAR: case GSQL_AGG_COUNT: case GSQL_AGG_SUM0:
        if (s.l) atomicAdd(reinterpret_cast<unsigned long long *>(&a.l[gid]), (unsigned long long)s.l);
        return;
    default: break;
    }
    if (!s.has) return;
    switch (a.kind) {
    case GSQL_AGG_SUM:
        if (a.in_type == GSQL_T_FP64) {
            atomicAdd(&a.d[gid], sa_d(s));
        } else {  // 128-bit: the low word's carry out goes into the high word's add
            const unsigned long long old = atomicAdd(reinterpret_cast<unsigned long long *>(&a.l[gid]), (unsigned long long)s.l);
            const unsigned long long hi = (unsigned long long)s.x + (old + (unsigned long long)s.l < old ? 1ULL : 0ULL);
            if (hi) atomicAdd(reinterpret_cast<unsigned long long *>(&a.hi[gid]), hi);
        }
        break;
    case GSQL_AGG_AVG: case GSQL_AGG_AVG_MERGE:
        atomicAdd(&a.d[gid], sa_d(s));
        atomicAdd(reinterpret_cast<unsigned long long *>(&a.l[gid]), (unsigned long long)s.l);
        break;
    case GSQL_AGG_MAX: atomicMax(reinterpret_cast<long long *>(&a.l[gid]), s.l); break;
    default: atomicMin(reinterpret_cast<long long *>(&a.l[gid]), s.l); break;  // MIN
    }
    a.has[gid] = 1;
}

// writeResultTo of a state: the value's words (hi: DEC128 only; DOUBLE as bits) and whether the result is NULL
// (SpecificType2DoubleAvgV2.java:70-84 for AVG: NULL without a row).
__device__ __forceinline__ bool state_result(int kind, int in_type, const SState &s, long long &lo, long long &hi) {
    lo = hi = 0;
    switch (kind) {
    case GSQL_AGG_COUNT_STAR: case GSQL_AGG_COUNT: case GSQL_AGG_SUM0: lo = s.l; return false;
    case GSQL_AGG_AVG: case GSQL_AGG_AVG_MERGE: {
        const bool ok = s.has && s.l != 0;
        if (ok) lo = __double_as_longlong(sa_d(s) / (double)s.l);
        return !ok;
    }
    default: break;
    }
    if (!s.has) return true;
    switch (kind) {
    case GSQL_AGG_SUM:
        if (in_type == GSQL_T_FP64) lo = s.x;
        else { lo = s.l; hi = s.x; }
        break;
    case GSQL_AGG_FIRST_VALUE: lo = s.l; break;  // INT32 sign-extended, INT64, or DOUBLE bits
    default:  // MIN / MAX
        lo = in_type == GSQL_T_FP64 ? __double_as_longlong(dbl_unsortable(s.l, kind == GSQL_AGG_MAX)) : s.l;
    }
    return false;
}

// ---- host side

// The state arrays a kind needs: words of l per group, whether hi and d exist, and the value l starts at.
struct AggStateArrays {
    int64_t l_words;
    bool hi, d;
    int64_t l_init;
};
static AggStateArrays agg_state_arrays(int kind, int in_type) {
    AggStateArrays r;
    r.l_words = kind == GSQL_AGG_FIRST_VALUE ? 2 : 1;  // one FvCell
    r.hi = kind == GSQL_AGG_SUM && in_type != GSQL_T_FP64;
    r.d = (kind == GSQL_AGG_SUM && in_type == GSQL_T_FP64) || kind == GSQL_AGG_AVG || kind == GSQL_AGG_AVG_MERGE;
    r.l_init = kind == GSQL_AGG_FIRST_VALUE ? -1 : state_zero(kind).l;  // both words of an FvCell: FV_EMPTY
    return r;
}

// The device view of call c (input type in_type) over the given state arrays (hi / d: null when the kind has none).
static AggDev agg_dev(const gsql_agg_call &c, int in_type, int64_t *l, int64_t *hi, double *d, uint8_t *has) {
    AggDev a;
    memset(&a, 0, sizeof(a));
    a.kind = c.kind;
    a.in_type = in_type;
    a.ncols = c.ncols;
    a.filter_col = c.filter_arg;
    for (int q = 0; q < 4; q++) a.cols[q] = c.cols[q];
    a.l = l;
    a.hi = hi;
    a.d = d;
    a.has = has;
    return a;
}
