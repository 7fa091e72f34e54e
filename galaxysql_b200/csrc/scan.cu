// scan.cu — vectorised Filter + Project behind gsql_scan_* (SURVEY §8f rank 1).
//
// Reference path replaced (EX/ = polardbx-executor/src/main/java/com/alibaba/polardbx/executor/):
//   EX/operator/VectorizedFilterExec.java (condition.eval -> selection array -> compacted chunk)
//   EX/operator/VectorizedProjectExec.java:40-143 (one VectorizedExpression per output column, evaluated per chunk)
//   EX/vectorized/** (the per-type expression classes: arithmetic, comparison, logic over Blocks with isNull[])
// Shape: ONE pass.  A block takes 1024-row tiles; every thread evaluates the filter program for its rows on a
// small typed stack (the program is uniform across threads: no divergence except NULL handling), the tile's
// survivors are ranked with warp ballots, one global cursor bump reserves their output range, and each survivor
// evaluates the output programs and writes its row.  Input columns are read once, surviving rows written once: the
// kernel is HBM-bound (input bytes + selectivity x output bytes); the interpreter costs ~10 warp-instructions per
// program step per 32 rows, far below the memory time.
#include <algorithm>
#include <vector>

#include "common.cuh"

namespace {

constexpr int SC_THREADS = 256;
constexpr int SC_RPT = 4;
constexpr int SC_TILE = SC_THREADS * SC_RPT;

struct DIns {        // device form of one instruction: operand types resolved on the host
    int16_t op;
    int8_t af, bf;   // operand a / b is a double (b = top of stack)
    int32_t arg;
    long long k;
};
struct DExpr {
    int32_t n, out_type;  // out_type: gsql_type of the result
    DIns ins[GSQL_MAX_EXPR_INS];
};
struct ScanDev {
    int32_t has_filter, n_out;
    DExpr filter;
    DExpr out[GSQL_MAX_SCAN_OUT];
};
struct ScanOut {
    void *data[GSQL_MAX_SCAN_OUT];
    uint8_t *nulls[GSQL_MAX_SCAN_OUT];
};

__device__ __forceinline__ double as_f(long long v, bool is_f) { return is_f ? __longlong_as_double(v) : (double)v; }

// CAST(double AS BIGINT / SIGNED) as the reference's CastToSigned, (long) Math.rint(d): round half to even, then Java's
// narrowing (saturating, NaN -> 0)
__device__ __forceinline__ long long java_rint_d2l(double d) {
    if (d != d) return 0;
    if (d >= 9223372036854775808.0) return 0x7fffffffffffffffLL;
    if (d <= -9223372036854775808.0) return (long long)0x8000000000000000ULL;
    return __double2ll_rn(d);
}

// Evaluates one program for the SC_RPT rows a thread owns in a tile (rows base + k * SC_THREADS), instruction by
// instruction: every program step is decoded ONCE and applied to the four rows, so the dispatch (the switch, the load of
// the instruction word) is amortised over them, and the four rows give every step four independent dependency chains.
// The operand stack lives in REGISTERS: four named slots per row that are shifted on push / pop (the program is uniform
// across the block, so the shifts are plain moves) — a stack indexed by a run-time pointer would sit in local memory.
// A row-at-a-time version of this interpreter was issue-bound on the per-row dispatch; programs deeper than 4 are rejected at create (GSQL_MAX_EXPR_STACK).
// live[k] == false rows are evaluated on row `base` (in bounds) and ignored by the caller.
struct EStack4 {
    long long v0[SC_RPT], v1[SC_RPT], v2[SC_RPT], v3[SC_RPT];
    bool n0[SC_RPT], n1[SC_RPT], n2[SC_RPT], n3[SC_RPT];
    __device__ __forceinline__ void push_down() {
#pragma unroll
        for (int k = 0; k < SC_RPT; k++) {
            v3[k] = v2[k]; n3[k] = n2[k];
            v2[k] = v1[k]; n2[k] = n1[k];
            v1[k] = v0[k]; n1[k] = n0[k];
        }
    }
    __device__ __forceinline__ void pop_up() {  // drops the top
#pragma unroll
        for (int k = 0; k < SC_RPT; k++) {
            v0[k] = v1[k]; n0[k] = n1[k];
            v1[k] = v2[k]; n1[k] = n2[k];
            v2[k] = v3[k]; n2[k] = n3[k];
        }
    }
};

// NULLS = false: no input column of the batch carries a NULL buffer and no program divides — every flag is a compile-time
// `false` and the flag bookkeeping (byte permutes, selects) disappears from the instruction stream.  A program with a DIV
// can make a NULL out of NULL-free inputs (zero divisor), so it always runs with NULLS = true.
// COND = true: the program may hold the conditional and set ops (GSQL_OP_CONST_NULL and up); IN and BETWEEN read their
// constants from `pool` (shared memory; each IN list sorted ascending by compile_expr).  COND = false compiles none of it.
template <bool NULLS, bool COND = false>
__device__ __forceinline__ void eval_expr4(const DExpr &E, const DColSet &in, int64_t base, const bool (&live)[SC_RPT], long long (&out)[SC_RPT],
                                           bool (&outnull)[SC_RPT], const long long *pool = nullptr) {
    EStack4 S;
#pragma unroll
    for (int k = 0; k < SC_RPT; k++) {
        S.v0[k] = S.v1[k] = S.v2[k] = S.v3[k] = 0;
        S.n0[k] = S.n1[k] = S.n2[k] = S.n3[k] = false;
    }
#pragma unroll 1
    for (int i = 0; i < E.n; i++) {
        const DIns I = E.ins[i];
        if constexpr (COND) {
            if (I.op >= GSQL_OP_CONST_NULL) {
                switch (I.op) {
                case GSQL_OP_CONST_NULL:
                    S.push_down();
#pragma unroll
                    for (int k = 0; k < SC_RPT; k++) { S.v0[k] = 0; S.n0[k] = NULLS; }
                    break;
                case GSQL_OP_CASE_WHEN:  // [acc, cond, then]: the first TRUE condition, compiled last, is applied last
#pragma unroll
                    for (int k = 0; k < SC_RPT; k++) {
                        const bool take = !(NULLS && S.n1[k]) && S.v1[k] != 0;
                        S.v2[k] = take ? S.v0[k] : S.v2[k];
                        S.n2[k] = NULLS && (take ? S.n0[k] : S.n2[k]);
                    }
                    S.pop_up();
                    S.pop_up();
                    break;
                case GSQL_OP_COALESCE:
#pragma unroll
                    for (int k = 0; k < SC_RPT; k++) {
                        const bool an = NULLS && S.n1[k];
                        S.v1[k] = an ? S.v0[k] : S.v1[k];
                        S.n1[k] = an && S.n0[k];
                    }
                    S.pop_up();
                    break;
                case GSQL_OP_BETWEEN: {
                    const long long lo = pool[I.arg], hi = pool[I.arg + 1];
#pragma unroll
                    for (int k = 0; k < SC_RPT; k++) {
                        const long long x = (NULLS && S.n0[k]) ? 0 : S.v0[k];
                        S.v0[k] = x >= lo && x <= hi;
                        S.n0[k] = false;
                    }
                    break;
                }
                default: {  // GSQL_OP_IN: lower bound in the sorted list pool[arg .. arg + k)
                    const int first = I.arg, end = I.arg + (int)I.k;
#pragma unroll
                    for (int k = 0; k < SC_RPT; k++) {
                        const long long x = (NULLS && S.n0[k]) ? 0 : S.v0[k];
                        int lo = first, hi = end;
                        while (lo < hi) {
                            const int mid = (lo + hi) >> 1;
                            if (pool[mid] < x) lo = mid + 1;
                            else hi = mid;
                        }
                        S.v0[k] = lo < end && pool[lo] == x;
                        S.n0[k] = false;
                    }
                    break;
                }
                }
                continue;
            }
        }
        switch (I.op) {
        case GSQL_OP_COL: {
            const DCol &c = in.c[I.arg];
            S.push_down();
            const bool is32 = c.type == GSQL_T_INT32;
#pragma unroll
            for (int k = 0; k < SC_RPT; k++) {
                const int64_t r = live[k] ? base + (int64_t)k * SC_THREADS : base;
                const bool n = NULLS && c.nulls != nullptr && c.nulls[r] != 0;
                long long v = is32 ? (long long)ld_stream_4(reinterpret_cast<const int *>(c.data) + r) : ld_stream_8(reinterpret_cast<const long long *>(c.data) + r);
                S.v0[k] = n ? 0 : v;
                S.n0[k] = n;
            }
            break;
        }
        case GSQL_OP_CONST_I64:
        case GSQL_OP_CONST_F64:
            S.push_down();
#pragma unroll
            for (int k = 0; k < SC_RPT; k++) { S.v0[k] = I.k; S.n0[k] = false; }
            break;
        case GSQL_OP_NEG:
#pragma unroll
            for (int k = 0; k < SC_RPT; k++)
                S.v0[k] = I.af ? __double_as_longlong(-__longlong_as_double(S.v0[k])) : (long long)(0ULL - (unsigned long long)S.v0[k]);
            break;
        case GSQL_OP_NOT:
#pragma unroll
            for (int k = 0; k < SC_RPT; k++) S.v0[k] = S.v0[k] == 0 ? 1 : 0;
            break;
        case GSQL_OP_IS_NULL:
#pragma unroll
            for (int k = 0; k < SC_RPT; k++) { S.v0[k] = (NULLS && S.n0[k]) ? 1 : 0; S.n0[k] = false; }
            break;
        case GSQL_OP_CAST_F64:
            if (!I.af) {
#pragma unroll
                for (int k = 0; k < SC_RPT; k++) S.v0[k] = __double_as_longlong((double)S.v0[k]);
            }
            break;
        case GSQL_OP_CAST_I64:
            if (I.af) {
#pragma unroll
                for (int k = 0; k < SC_RPT; k++) S.v0[k] = java_rint_d2l(__longlong_as_double(S.v0[k]));
            }
            break;
        case GSQL_OP_AND:
        case GSQL_OP_OR: {  // SQL three-valued logic
            const bool is_and = I.op == GSQL_OP_AND;
#pragma unroll
            for (int k = 0; k < SC_RPT; k++) {
                const long long b = S.v0[k], a = S.v1[k];
                const bool bn = NULLS && S.n0[k], an = NULLS && S.n1[k];
                if (is_and) {
                    const bool f = (!an && a == 0) || (!bn && b == 0);
                    S.v1[k] = f ? 0 : 1;
                    S.n1[k] = !f && (an || bn);
                } else {
                    const bool t = (!an && a != 0) || (!bn && b != 0);
                    S.v1[k] = t ? 1 : 0;
                    S.n1[k] = !t && (an || bn);
                }
            }
            S.pop_up();
            break;
        }
        default: {  // binary arithmetic / comparison: a = second slot, b = top
            const bool fl = I.af || I.bf || I.op == GSQL_OP_DIV;
#pragma unroll
            for (int k = 0; k < SC_RPT; k++) {
                const long long b = S.v0[k], a = S.v1[k];
                bool n = NULLS && (S.n0[k] || S.n1[k]);
                long long res = 0;
                if (fl) {
                    const double x = as_f(a, I.af), y = as_f(b, I.bf);
                    switch (I.op) {
                    case GSQL_OP_ADD: res = __double_as_longlong(x + y); break;
                    case GSQL_OP_SUB: res = __double_as_longlong(x - y); break;
                    case GSQL_OP_MUL: res = __double_as_longlong(x * y); break;
                    case GSQL_OP_DIV:  // a zero divisor (0, 0.0, -0.0; not NaN) makes the quotient NULL, as the reference's Divide
                        res = __double_as_longlong(x / y);
                        n = n || (NULLS && y == 0.0);
                        break;
                    case GSQL_OP_LT: res = x < y; break;
                    case GSQL_OP_LE: res = x <= y; break;
                    case GSQL_OP_GT: res = x > y; break;
                    case GSQL_OP_GE: res = x >= y; break;
                    case GSQL_OP_EQ: res = x == y; break;
                    default: res = x != y; break;
                    }
                } else {
                    switch (I.op) {
                    case GSQL_OP_ADD: res = (long long)((unsigned long long)a + (unsigned long long)b); break;
                    case GSQL_OP_SUB: res = (long long)((unsigned long long)a - (unsigned long long)b); break;
                    case GSQL_OP_MUL: res = (long long)((unsigned long long)a * (unsigned long long)b); break;
                    case GSQL_OP_LT: res = a < b; break;
                    case GSQL_OP_LE: res = a <= b; break;
                    case GSQL_OP_GT: res = a > b; break;
                    case GSQL_OP_GE: res = a >= b; break;
                    case GSQL_OP_EQ: res = a == b; break;
                    default: res = a != b; break;
                    }
                }
                S.v1[k] = n ? 0 : res;
                S.n1[k] = n;
            }
            S.pop_up();
            break;
        }
        }
    }
#pragma unroll
    for (int k = 0; k < SC_RPT; k++) { out[k] = S.v0[k]; outnull[k] = NULLS && S.n0[k]; }
}

template <bool NULLS, bool COND>
__device__ __forceinline__ void scan_tiles(const ScanDev *__restrict__ S, const DColSet &in, int64_t rows, const ScanOut &O, unsigned long long *cursor,
                                           int32_t *flags, const long long *pool) {
    __shared__ unsigned int wcount[SC_THREADS / 32][SC_RPT];
    __shared__ unsigned long long tile_base;
    const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
    const int64_t ntiles = (rows + SC_TILE - 1) / SC_TILE;
    for (int64_t tile = blockIdx.x; tile < ntiles; tile += gridDim.x) {
        const int64_t t0 = tile * SC_TILE;
        const int64_t base = t0 + threadIdx.x;  // row of slot 0 (always < rows for the threads of a started tile? no: guarded below)
        bool pass[SC_RPT];
        unsigned int ballot[SC_RPT];
#pragma unroll
        for (int k = 0; k < SC_RPT; k++) pass[k] = t0 + k * SC_THREADS + threadIdx.x < rows;
        const int64_t safe = base < rows ? base : rows - 1;  // dead slots re-read an in-bounds row
        if (S->has_filter) {
            long long fv[SC_RPT];
            bool fn[SC_RPT];
            eval_expr4<NULLS, COND>(S->filter, in, safe, pass, fv, fn, pool);
#pragma unroll
            for (int k = 0; k < SC_RPT; k++) pass[k] = pass[k] && !fn[k] && fv[k] != 0;
        }
#pragma unroll
        for (int k = 0; k < SC_RPT; k++) {
            ballot[k] = __ballot_sync(0xffffffffu, pass[k]);
            if (lane == 0) wcount[warp][k] = __popc(ballot[k]);
        }
        __syncthreads();
        if (warp == 0) {  // 32 cells: exclusive scan in (slot k, warp) order keeps the tile's rows in input order
            const int k = lane / (SC_THREADS / 32), w = lane % (SC_THREADS / 32);
            const unsigned int c = wcount[w][k];
            unsigned int incl = c;
#pragma unroll
            for (int d = 1; d < 32; d <<= 1) {
                const unsigned int t = __shfl_up_sync(0xffffffffu, incl, d);
                if (lane >= d) incl += t;
            }
            const unsigned int total = __shfl_sync(0xffffffffu, incl, 31);
            wcount[w][k] = incl - c;
            if (lane == 0) tile_base = total ? atomicAdd(cursor, (unsigned long long)total) : 0ULL;
            static_assert((SC_THREADS / 32) * SC_RPT == 32, "cell scan assumes 32 cells");
        }
        __syncthreads();
        unsigned long long pos[SC_RPT];
#pragma unroll
        for (int k = 0; k < SC_RPT; k++) pos[k] = tile_base + wcount[warp][k] + __popc(ballot[k] & ((1u << lane) - 1u));
        for (int e = 0; e < S->n_out; e++) {
            long long v[SC_RPT];
            bool n[SC_RPT];
            eval_expr4<NULLS, COND>(S->out[e], in, safe, pass, v, n, pool);
            const bool is32 = S->out[e].out_type == GSQL_T_INT32;
#pragma unroll
            for (int k = 0; k < SC_RPT; k++) {
                if (!pass[k]) continue;
                if (O.nulls[e]) O.nulls[e][pos[k]] = n[k] ? 1 : 0;
                else if (n[k]) flags[0] = 1;
                if (is32) reinterpret_cast<int *>(O.data[e])[pos[k]] = (int)v[k];
                else reinterpret_cast<long long *>(O.data[e])[pos[k]] = v[k];
            }
        }
        __syncthreads();  // wcount / tile_base are rewritten by the next tile
    }
}

template <bool NULLS>
__global__ void __launch_bounds__(SC_THREADS) k_scan(const ScanDev *__restrict__ S, const __grid_constant__ DColSet in, int64_t rows,
                                                     const __grid_constant__ ScanOut O, unsigned long long *cursor, int32_t *flags) {
    scan_tiles<NULLS, false>(S, in, rows, O, cursor, flags, nullptr);
}

// Programs with the conditional and set ops (gsql_scan_create2): the same tiles; the constant pool is staged in shared memory.
template <bool NULLS>
__global__ void __launch_bounds__(SC_THREADS) k_scan_cond(const ScanDev *__restrict__ S, const __grid_constant__ DColSet in, int64_t rows,
                                                          const __grid_constant__ ScanOut O, unsigned long long *cursor, int32_t *flags,
                                                          const long long *__restrict__ pool, int32_t npool) {
    __shared__ long long spool[GSQL_MAX_SCAN_POOL];
    for (int i = threadIdx.x; i < npool; i += SC_THREADS) spool[i] = pool[i];
    __syncthreads();
    scan_tiles<NULLS, true>(S, in, rows, O, cursor, flags, spool);
}

// ---------------------------------------------------------------------------------------------- specialised shapes
// The programs the MPP plans actually send are tiny: a filter `column <cmp> constant` over an integer column and outputs
// that are either a column or `a * (1 - b)` over two DOUBLE columns (TPC-H Q3: scan_c / scan_o / scan_l of
// galaxysql_b200/pipelines.py).  The host recognises that shape at create (scan_fast_plan) and, for a batch without NULL
// buffers, runs k_scan_fast: the same tile structure and output order as k_scan, but the filter is an interval test and
// the outputs are straight-line code — several times fewer thread-instructions per row than the issue-bound
// interpreter.  Everything else (deeper programs, NULL buffers) stays on k_scan.
struct FastOut {
    int32_t kind;  // 0: column a; 1: a * (1.0 - b) (both DOUBLE)
    int32_t a, b;
    int32_t w;     // output width in bytes (4 or 8)
};
struct ScanFastPlan {
    int32_t ok, has_filter, fcol, fneg;  // filter: pass = (lo <= x && x <= hi) != fneg
    int64_t lo, hi;
    int32_t n_out, pad;
    FastOut out[GSQL_MAX_SCAN_OUT];
};

// `column IN (list)`: a 64-bit mask over [base, base + 64) when the list spans fewer than 64 values, otherwise a lower-bound
// search in the sorted list, staged in shared memory.
struct FastSet {
    int32_t kind, n;  // kind: -1 none, 0 mask, 1 sorted search (n entries of the scan's device pool from `at`)
    int32_t at, pad;
    long long base;
    unsigned long long mask;
};

// The filter of a specialised shape tests one integer column: SET = 0 the interval of F (k_scan_fast), 1 the mask of T,
// 2 a search in the sorted `list` of T.n entries (k_scan_fast_set).
template <int SET>
__device__ __forceinline__ void scan_fast_tiles(const ScanFastPlan &F, const DColSet &in, int64_t rows, const ScanOut &O, unsigned long long *cursor,
                                                const FastSet *T, const long long *list) {
    __shared__ unsigned int wcount[SC_THREADS / 32][SC_RPT];
    __shared__ unsigned long long tile_base;
    const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
    const int64_t ntiles = (rows + SC_TILE - 1) / SC_TILE;
    for (int64_t tile = blockIdx.x; tile < ntiles; tile += gridDim.x) {
        const int64_t t0 = tile * SC_TILE + threadIdx.x;  // this thread's row in slot 0; slot k is k * SC_THREADS further
        bool pass[SC_RPT];
        unsigned int ballot[SC_RPT];
#pragma unroll
        for (int k = 0; k < SC_RPT; k++) pass[k] = t0 + k * SC_THREADS < rows;
        if (F.has_filter) {
            const DCol &c = in.c[F.fcol];
            long long x[SC_RPT];
            if (c.type == GSQL_T_INT32) {
#pragma unroll
                for (int k = 0; k < SC_RPT; k++) x[k] = pass[k] ? (long long)ld_stream_4(reinterpret_cast<const int *>(c.data) + t0 + k * SC_THREADS) : 0;
            } else {
#pragma unroll
                for (int k = 0; k < SC_RPT; k++) x[k] = pass[k] ? ld_stream_8(reinterpret_cast<const long long *>(c.data) + t0 + k * SC_THREADS) : 0;
            }
#pragma unroll
            for (int k = 0; k < SC_RPT; k++) {
                if constexpr (SET == 0) {
                    pass[k] = pass[k] && ((x[k] >= F.lo && x[k] <= F.hi) != (F.fneg != 0));
                } else if constexpr (SET == 1) {
                    const unsigned long long d = (unsigned long long)x[k] - (unsigned long long)T->base;
                    pass[k] = pass[k] && d < 64 && ((T->mask >> d) & 1ULL);
                } else {
                    int lo = 0, hi = T->n;
                    while (lo < hi) {
                        const int mid = (lo + hi) >> 1;
                        if (list[mid] < x[k]) lo = mid + 1;
                        else hi = mid;
                    }
                    pass[k] = pass[k] && lo < T->n && list[lo] == x[k];
                }
            }
        }
#pragma unroll
        for (int k = 0; k < SC_RPT; k++) {
            ballot[k] = __ballot_sync(0xffffffffu, pass[k]);
            if (lane == 0) wcount[warp][k] = __popc(ballot[k]);
        }
        __syncthreads();
        if (warp == 0) {  // 32 cells: exclusive scan in (slot k, warp) order keeps the tile's rows in input order
            const int k = lane / (SC_THREADS / 32), w = lane % (SC_THREADS / 32);
            const unsigned int c = wcount[w][k];
            unsigned int incl = c;
#pragma unroll
            for (int d = 1; d < 32; d <<= 1) {
                const unsigned int t = __shfl_up_sync(0xffffffffu, incl, d);
                if (lane >= d) incl += t;
            }
            const unsigned int total = __shfl_sync(0xffffffffu, incl, 31);
            wcount[w][k] = incl - c;
            if (lane == 0) tile_base = total ? atomicAdd(cursor, (unsigned long long)total) : 0ULL;
        }
        __syncthreads();
        unsigned long long pos[SC_RPT];
#pragma unroll
        for (int k = 0; k < SC_RPT; k++) pos[k] = tile_base + wcount[warp][k] + __popc(ballot[k] & ((1u << lane) - 1u));
#pragma unroll 1
        for (int e = 0; e < F.n_out; e++) {
            const FastOut o = F.out[e];
            const DCol &ca = in.c[o.a];
            if (o.kind == 1) {
                const DCol &cb = in.c[o.b];
                double va[SC_RPT], vb[SC_RPT];
#pragma unroll
                for (int k = 0; k < SC_RPT; k++) {
                    va[k] = pass[k] ? __longlong_as_double(ld_stream_8(reinterpret_cast<const long long *>(ca.data) + t0 + k * SC_THREADS)) : 0.0;
                    vb[k] = pass[k] ? __longlong_as_double(ld_stream_8(reinterpret_cast<const long long *>(cb.data) + t0 + k * SC_THREADS)) : 0.0;
                }
#pragma unroll
                for (int k = 0; k < SC_RPT; k++)
                    if (pass[k]) reinterpret_cast<double *>(O.data[e])[pos[k]] = va[k] * (1.0 - vb[k]);
            } else if (o.w == 4) {
                int v[SC_RPT];
#pragma unroll
                for (int k = 0; k < SC_RPT; k++) v[k] = pass[k] ? ld_stream_4(reinterpret_cast<const int *>(ca.data) + t0 + k * SC_THREADS) : 0;
#pragma unroll
                for (int k = 0; k < SC_RPT; k++)
                    if (pass[k]) reinterpret_cast<int *>(O.data[e])[pos[k]] = v[k];
            } else {
                long long v[SC_RPT];
#pragma unroll
                for (int k = 0; k < SC_RPT; k++) v[k] = pass[k] ? ld_stream_8(reinterpret_cast<const long long *>(ca.data) + t0 + k * SC_THREADS) : 0;
#pragma unroll
                for (int k = 0; k < SC_RPT; k++)
                    if (pass[k]) reinterpret_cast<long long *>(O.data[e])[pos[k]] = v[k];
            }
            if (O.nulls[e]) {
#pragma unroll
                for (int k = 0; k < SC_RPT; k++)
                    if (pass[k]) O.nulls[e][pos[k]] = 0;
            }
        }
        __syncthreads();  // wcount / tile_base are rewritten by the next tile
    }
}

__global__ void __launch_bounds__(SC_THREADS) k_scan_fast(const __grid_constant__ ScanFastPlan F, const __grid_constant__ DColSet in, int64_t rows,
                                                          const __grid_constant__ ScanOut O, unsigned long long *cursor) {
    scan_fast_tiles<0>(F, in, rows, O, cursor, nullptr, nullptr);
}

template <bool SEARCH>
__global__ void __launch_bounds__(SC_THREADS) k_scan_fast_set(const __grid_constant__ ScanFastPlan F, const __grid_constant__ FastSet T,
                                                              const __grid_constant__ DColSet in, int64_t rows, const __grid_constant__ ScanOut O,
                                                              unsigned long long *cursor, const long long *__restrict__ pool) {
    __shared__ long long list[SEARCH ? GSQL_MAX_IN_LIST : 1];
    if constexpr (SEARCH) {
        for (int i = threadIdx.x; i < T.n; i += SC_THREADS) list[i] = pool[T.at + i];
        __syncthreads();
    }
    scan_fast_tiles<SEARCH ? 2 : 1>(F, in, rows, O, cursor, &T, list);
}

// Recognises the specialised shape in the caller's programs (host, at create).  in_types: the scan's input column types.
// fd / dpool: the compiled filter and the device pool its IN / BETWEEN constants were copied to (each IN list sorted).
static void scan_fast_plan(ScanFastPlan *Fp, FastSet *T, const gsql_scan_spec &s, const int32_t *out_types, const DExpr &fd,
                           const std::vector<long long> &dpool) {
    ScanFastPlan &F = *Fp;
    memset(&F, 0, sizeof(F));
    memset(T, 0, sizeof(*T));
    T->kind = -1;
    int no_fast = 0;
    if (env_knob("GSQL_SCAN_NO_FAST", &no_fast) && no_fast) return;
    auto is_col = [&](const gsql_expr_ins &I) { return I.op == GSQL_OP_COL && I.arg >= 0 && I.arg < s.n_input_cols; };
    if (s.has_filter && s.filter.n == 2 && is_col(s.filter.ins[0]) && s.input_types[s.filter.ins[0].arg] != GSQL_T_FP64 &&
        (s.filter.ins[1].op == GSQL_OP_BETWEEN || s.filter.ins[1].op == GSQL_OP_IN)) {  // COL c, BETWEEN / IN over an integer column
        const DIns &d = fd.ins[1];
        F.has_filter = 1;
        F.fcol = s.filter.ins[0].arg;
        if (d.op == GSQL_OP_BETWEEN) {  // the interval test of k_scan_fast
            F.lo = dpool[d.arg];
            F.hi = dpool[d.arg + 1];
        } else if ((unsigned long long)dpool[d.arg + d.k - 1] - (unsigned long long)dpool[d.arg] < 64) {
            T->kind = 0;
            T->base = dpool[d.arg];
            for (int i = 0; i < (int)d.k; i++) T->mask |= 1ULL << ((unsigned long long)dpool[d.arg + i] - (unsigned long long)T->base);
        } else {
            T->kind = 1;
            T->at = d.arg;
            T->n = (int32_t)d.k;
        }
    } else if (s.has_filter) {  // COL c, CONST_I64 k, <cmp>  ==  c <cmp> k over an integer column
        const gsql_expr &f = s.filter;
        if (f.n != 3 || !is_col(f.ins[0]) || f.ins[1].op != GSQL_OP_CONST_I64) return;
        if (s.input_types[f.ins[0].arg] == GSQL_T_FP64) return;
        const int64_t v = f.ins[1].k.i, mn = INT64_MIN, mx = INT64_MAX;
        F.has_filter = 1;
        F.fcol = f.ins[0].arg;
        F.lo = mn; F.hi = mx; F.fneg = 0;
        switch (f.ins[2].op) {
        case GSQL_OP_LE: F.hi = v; break;
        case GSQL_OP_LT: if (v == mn) { F.lo = 1; F.hi = 0; } else F.hi = v - 1; break;
        case GSQL_OP_GE: F.lo = v; break;
        case GSQL_OP_GT: if (v == mx) { F.lo = 1; F.hi = 0; } else F.lo = v + 1; break;
        case GSQL_OP_EQ: F.lo = F.hi = v; break;
        case GSQL_OP_NE: F.lo = F.hi = v; F.fneg = 1; break;
        default: return;
        }
    }
    F.n_out = s.n_out;
    for (int e = 0; e < s.n_out; e++) {
        const gsql_expr &x = s.out[e];
        FastOut &o = F.out[e];
        if (x.n == 1 && is_col(x.ins[0])) {  // a column, as it is
            o.kind = 0;
            o.a = o.b = x.ins[0].arg;
            o.w = s.input_types[o.a] == GSQL_T_INT32 ? 4 : 8;
            if (out_types[e] != s.input_types[o.a]) return;
        } else if (x.n == 5 && is_col(x.ins[0]) && x.ins[1].op == GSQL_OP_CONST_F64 && x.ins[1].k.d == 1.0 && is_col(x.ins[2]) &&
                   x.ins[3].op == GSQL_OP_SUB && x.ins[4].op == GSQL_OP_MUL && s.input_types[x.ins[0].arg] == GSQL_T_FP64 &&
                   s.input_types[x.ins[2].arg] == GSQL_T_FP64) {  // COL a, 1.0, COL b, SUB, MUL  ==  a * (1.0 - b)
            o.kind = 1;
            o.a = x.ins[0].arg;
            o.b = x.ins[2].arg;
            o.w = 8;
        } else {
            return;
        }
    }
    F.ok = 1;
}

// The caller's constant pool, for programs of gsql_scan_create2 (cond: the ops from GSQL_OP_CONST_NULL on are accepted).
// compile_expr copies each IN list (sorted) and BETWEEN pair into dpool, the pool the kernels read, and points arg there.
struct PoolIn {
    bool cond;
    const int64_t *pool;
    int32_t npool;
    std::vector<long long> *dpool;
    bool *has_null;  // set if a program pushes a NULL constant: NULLs then appear in NULL-free batches
};

// Host: type-checks a program, fills the device form.  Returns the result type or -1; sets *has_div if the program divides.
int compile_expr(const gsql_expr &E, const int32_t *in_types, int n_in, DExpr *D, bool *has_div, char *err, size_t errn, const PoolIn &P) {
    if (E.n < 1 || E.n > GSQL_MAX_EXPR_INS) { snprintf(err, errn, "program length %d", E.n); return -1; }
    bool isf[GSQL_MAX_EXPR_STACK];
    int sp = 0;
    D->n = E.n;
    for (int i = 0; i < E.n; i++) {
        const gsql_expr_ins &I = E.ins[i];
        DIns &d = D->ins[i];
        d.op = (int16_t)I.op;
        d.af = d.bf = 0;
        d.arg = I.arg;
        d.k = I.k.i;
        switch (I.op) {
        case GSQL_OP_COL:
            if (I.arg < 0 || I.arg >= n_in) { snprintf(err, errn, "column %d out of range", I.arg); return -1; }
            if (sp >= GSQL_MAX_EXPR_STACK) { snprintf(err, errn, "stack deeper than %d", GSQL_MAX_EXPR_STACK); return -1; }
            isf[sp++] = in_types[I.arg] == GSQL_T_FP64;
            break;
        case GSQL_OP_CONST_I64:
        case GSQL_OP_CONST_F64:
            if (sp >= GSQL_MAX_EXPR_STACK) { snprintf(err, errn, "stack deeper than %d", GSQL_MAX_EXPR_STACK); return -1; }
            isf[sp++] = I.op == GSQL_OP_CONST_F64;
            break;
        case GSQL_OP_NEG: case GSQL_OP_NOT: case GSQL_OP_IS_NULL: case GSQL_OP_CAST_F64: case GSQL_OP_CAST_I64:
            if (sp < 1) { snprintf(err, errn, "stack underflow at %d", i); return -1; }
            d.af = isf[sp - 1];
            if (I.op == GSQL_OP_NOT && isf[sp - 1]) { snprintf(err, errn, "NOT over a double"); return -1; }
            if (I.op == GSQL_OP_IS_NULL || I.op == GSQL_OP_CAST_I64 || I.op == GSQL_OP_NOT) isf[sp - 1] = false;
            if (I.op == GSQL_OP_CAST_F64) isf[sp - 1] = true;
            break;
        case GSQL_OP_ADD: case GSQL_OP_SUB: case GSQL_OP_MUL: case GSQL_OP_DIV:
        case GSQL_OP_LT: case GSQL_OP_LE: case GSQL_OP_GT: case GSQL_OP_GE: case GSQL_OP_EQ: case GSQL_OP_NE:
        case GSQL_OP_AND: case GSQL_OP_OR:
            if (sp < 2) { snprintf(err, errn, "stack underflow at %d", i); return -1; }
            d.af = isf[sp - 2];
            d.bf = isf[sp - 1];
            if ((I.op == GSQL_OP_AND || I.op == GSQL_OP_OR) && (d.af || d.bf)) { snprintf(err, errn, "AND/OR over a double"); return -1; }
            sp--;
            if (I.op == GSQL_OP_DIV) *has_div = true;
            if (I.op >= GSQL_OP_LT) isf[sp - 1] = false;                       // comparisons / logic -> BIGINT 0/1
            else isf[sp - 1] = d.af || d.bf || I.op == GSQL_OP_DIV;
            break;
        case GSQL_OP_CONST_NULL:
            if (!P.cond) { snprintf(err, errn, "unknown op %d", I.op); return -1; }
            if (I.arg != GSQL_T_INT64 && I.arg != GSQL_T_FP64) { snprintf(err, errn, "NULL of type %d", I.arg); return -1; }
            if (sp >= GSQL_MAX_EXPR_STACK) { snprintf(err, errn, "stack deeper than %d", GSQL_MAX_EXPR_STACK); return -1; }
            isf[sp++] = I.arg == GSQL_T_FP64;
            *P.has_null = true;
            break;
        case GSQL_OP_CASE_WHEN:
            if (!P.cond) { snprintf(err, errn, "unknown op %d", I.op); return -1; }
            if (sp < 3) { snprintf(err, errn, "stack underflow at %d", i); return -1; }
            if (isf[sp - 2]) { snprintf(err, errn, "CASE condition is a double"); return -1; }
            if (isf[sp - 3] != isf[sp - 1]) { snprintf(err, errn, "CASE branches of two types"); return -1; }
            sp -= 2;
            break;
        case GSQL_OP_COALESCE:
            if (!P.cond) { snprintf(err, errn, "unknown op %d", I.op); return -1; }
            if (sp < 2) { snprintf(err, errn, "stack underflow at %d", i); return -1; }
            if (isf[sp - 2] != isf[sp - 1]) { snprintf(err, errn, "COALESCE of two types"); return -1; }
            sp--;
            break;
        case GSQL_OP_BETWEEN:
        case GSQL_OP_IN: {
            if (!P.cond) { snprintf(err, errn, "unknown op %d", I.op); return -1; }
            if (sp < 1) { snprintf(err, errn, "stack underflow at %d", i); return -1; }
            if (isf[sp - 1]) { snprintf(err, errn, "IN / BETWEEN over a double"); return -1; }
            const int64_t cnt = I.op == GSQL_OP_BETWEEN ? 2 : I.k.i;
            if (cnt < 1 || cnt > GSQL_MAX_IN_LIST) { snprintf(err, errn, "IN list of %lld", (long long)cnt); return -1; }
            if (I.arg < 0 || (int64_t)I.arg + cnt > P.npool) { snprintf(err, errn, "pool range %d+%lld outside %d", I.arg, (long long)cnt, P.npool); return -1; }
            if ((int64_t)P.dpool->size() + cnt > GSQL_MAX_SCAN_POOL) { snprintf(err, errn, "more than %d pool entries", GSQL_MAX_SCAN_POOL); return -1; }
            d.arg = (int32_t)P.dpool->size();
            d.k = cnt;
            P.dpool->insert(P.dpool->end(), P.pool + I.arg, P.pool + I.arg + cnt);
            if (I.op == GSQL_OP_IN) std::sort(P.dpool->begin() + d.arg, P.dpool->end());
            break;
        }
        default:
            snprintf(err, errn, "unknown op %d", I.op);
            return -1;
        }
    }
    if (sp != 1) { snprintf(err, errn, "program leaves %d values", sp); return -1; }
    int t = isf[0] ? GSQL_T_FP64 : GSQL_T_INT64;
    if (E.n == 1 && E.ins[0].op == GSQL_OP_COL) t = in_types[E.ins[0].arg];  // pass-through keeps the column's type
    D->out_type = t;
    return t;
}

}  // namespace

struct gsql_scan {
    gsql_ctx *ctx;
    gsql_scan_spec spec;
    ScanDev host;
    DevBuf dev, cursor, flags;
    int32_t out_types[GSQL_MAX_SCAN_OUT];
    ScanFastPlan fast;  // fast.ok: the programs have the specialised shape (k_scan_fast for NULL-free batches)
    FastSet fset;       // fset.kind >= 0: the fast filter is an IN list (k_scan_fast_set)
    bool has_div;       // some program divides: NULLs can appear in a NULL-free batch, so k_scan<false> is never used
    bool has_null;      // some program pushes a NULL constant: likewise
    bool has_cond;      // some program holds an op from GSQL_OP_CONST_NULL on: k_scan_cond
    int32_t npool;      // entries of `pool`, the device pool (IN lists sorted)
    DevBuf pool;
};

static gsql_status scan_create(gsql_ctx *ctx, const gsql_scan_spec *spec, bool cond, const int64_t *pool, int32_t npool, gsql_scan **out) {
    if (!ctx || !spec || !out) return GSQL_E_INVALID;
    if (ctx->sticky) return GSQL_E_CUDA;
    *out = nullptr;
    const gsql_scan_spec &s = *spec;
    if (s.n_input_cols < 1 || s.n_input_cols > GSQL_MAX_COLS || s.n_out < 1 || s.n_out > GSQL_MAX_SCAN_OUT)
        return gsql_set_error(ctx, GSQL_E_INVALID, "bad scan spec sizes");
    for (int i = 0; i < s.n_input_cols; i++)
        if (s.input_types[i] < GSQL_T_INT32 || s.input_types[i] > GSQL_T_FP64) return gsql_set_error(ctx, GSQL_E_UNSUPPORTED, "input col %d type", i);
    gsql_scan *sc = new gsql_scan();
    sc->ctx = ctx;
    sc->spec = s;
    memset(&sc->host, 0, sizeof(sc->host));
    char err[128] = {0};
    sc->host.has_filter = s.has_filter != 0;
    sc->host.n_out = s.n_out;
    sc->has_div = sc->has_null = false;
    std::vector<long long> dpool;
    const PoolIn P{cond, pool, npool, &dpool, &sc->has_null};
    if (s.has_filter) {
        int t = compile_expr(s.filter, s.input_types, s.n_input_cols, &sc->host.filter, &sc->has_div, err, sizeof(err), P);
        if (t < 0 || t == GSQL_T_FP64) {
            delete sc;
            return gsql_set_error(ctx, GSQL_E_INVALID, "filter: %s", t < 0 ? err : "must be an integer / boolean expression");
        }
    }
    for (int e = 0; e < s.n_out; e++) {
        int t = compile_expr(s.out[e], s.input_types, s.n_input_cols, &sc->host.out[e], &sc->has_div, err, sizeof(err), P);
        if (t < 0) { delete sc; return gsql_set_error(ctx, GSQL_E_INVALID, "output %d: %s", e, err); }
        sc->out_types[e] = t;
    }
    sc->has_cond = false;
    for (int e = -1; e < s.n_out; e++) {
        const gsql_expr &x = e < 0 ? s.filter : s.out[e];
        if (e < 0 && !s.has_filter) continue;
        for (int i = 0; i < x.n; i++) sc->has_cond |= x.ins[i].op >= GSQL_OP_CONST_NULL;
    }
    scan_fast_plan(&sc->fast, &sc->fset, s, sc->out_types, sc->host.filter, dpool);
    sc->npool = (int32_t)dpool.size();
    cudaSetDevice(ctx->device);
    gsql_status st = sc->dev.alloc(ctx, sizeof(ScanDev));
    if (st == GSQL_OK && sc->npool) st = sc->pool.alloc(ctx, dpool.size() * sizeof(long long));
    if (st == GSQL_OK && sc->npool &&
        cudaMemcpyAsync(sc->pool.p, dpool.data(), dpool.size() * sizeof(long long), cudaMemcpyHostToDevice, ctx->stream) != cudaSuccess)
        st = GSQL_E_CUDA;
    if (st == GSQL_OK) st = sc->cursor.alloc(ctx, 16);
    if (st == GSQL_OK) st = sc->flags.alloc(ctx, 16);
    if (st == GSQL_OK && cudaMemcpyAsync(sc->dev.p, &sc->host, sizeof(ScanDev), cudaMemcpyHostToDevice, ctx->stream) != cudaSuccess) st = GSQL_E_CUDA;
    if (st == GSQL_OK && cudaMemsetAsync(sc->flags.p, 0, 16, ctx->stream) != cudaSuccess) st = GSQL_E_CUDA;
    if (st == GSQL_OK && cudaStreamSynchronize(ctx->stream) != cudaSuccess) st = GSQL_E_CUDA;  // `host` may go away with the handle
    if (st != GSQL_OK) { delete sc; return st; }
    gsql_ctx_retain(ctx);
    *out = sc;
    return GSQL_OK;
}

extern "C" gsql_status gsql_scan_create(gsql_ctx *ctx, const gsql_scan_spec *spec, gsql_scan **out) {
    return scan_create(ctx, spec, false, nullptr, 0, out);
}

extern "C" gsql_status gsql_scan_create2(gsql_ctx *ctx, const gsql_scan_spec *spec, const int64_t *pool, int32_t npool, gsql_scan **out) {
    if (npool < 0 || npool > GSQL_MAX_SCAN_POOL || (npool > 0 && !pool)) {
        if (!ctx || !out) return GSQL_E_INVALID;
        *out = nullptr;
        return gsql_set_error(ctx, GSQL_E_INVALID, "constant pool of %d entries", npool);
    }
    return scan_create(ctx, spec, true, pool, npool, out);
}

extern "C" void gsql_scan_destroy(gsql_scan *s) { destroy_handle(s); }

extern "C" gsql_status gsql_scan_output_schema(gsql_scan *s, int32_t *ncols, int32_t *types) {
    if (!s || !ncols) return GSQL_E_INVALID;
    return output_schema(s->spec.n_out, s->out_types, ncols, types);
}

extern "C" gsql_status gsql_scan_apply(gsql_scan *s, const gsql_batch *in, gsql_batch *out, int64_t out_capacity, int64_t *out_rows) {
    if (!s || !in || !out || !out_rows) return GSQL_E_INVALID;
    gsql_ctx *ctx = s->ctx;
    if (ctx->sticky) return GSQL_E_CUDA;
    const gsql_scan_spec &sp = s->spec;
    GSQL_TRY(validate_batch(ctx, in, sp.n_input_cols, sp.input_types));
    GSQL_TRY(validate_batch(ctx, out, sp.n_out, s->out_types));
    if (in->mem != out->mem) return gsql_set_error(ctx, GSQL_E_INVALID, "in and out must live in the same memory space");
    *out_rows = 0;
    out->rows = 0;
    if (in->rows == 0) return GSQL_OK;
    if (out_capacity < in->rows) {
        *out_rows = in->rows;
        return gsql_set_error(ctx, GSQL_E_CAPACITY, "scan output must hold the input's %lld rows", (long long)in->rows);
    }
    GSQL_CUDA(ctx, cudaSetDevice(ctx->device));
    StagedBatch sb;
    GSQL_TRY(stage_batch(ctx, in, &sb));
    const DColSet cols = sb.set();
    OutBinding ob;
    GSQL_TRY(out_bind(ctx, out, in->rows, &ob));
    ScanOut O;
    memset(&O, 0, sizeof(O));
    for (int e = 0; e < sp.n_out; e++) {
        O.data[e] = ob.data[e];
        O.nulls[e] = ob.nulls[e];
    }
    GSQL_CUDA(ctx, cudaMemsetAsync(s->cursor.p, 0, 16, ctx->stream));
    {
        KernelScope ks(ctx, "scan_filter_project");
        int64_t tiles = div_up(in->rows, SC_TILE);
        int64_t g = tiles < (int64_t)ctx->sm_count * 8 ? tiles : (int64_t)ctx->sm_count * 8;
        bool any_mask = false;
        for (int i = 0; i < sb.ncols; i++) any_mask |= sb.cols[i].nulls != nullptr;
        const long long *pool = reinterpret_cast<const long long *>(s->pool.p);
        if (!any_mask && s->fast.ok && s->fset.kind == 0)
            k_scan_fast_set<false><<<(int)g, SC_THREADS, 0, ctx->stream>>>(s->fast, s->fset, cols, in->rows, O, s->cursor.as<unsigned long long>(), pool);
        else if (!any_mask && s->fast.ok && s->fset.kind == 1)
            k_scan_fast_set<true><<<(int)g, SC_THREADS, 0, ctx->stream>>>(s->fast, s->fset, cols, in->rows, O, s->cursor.as<unsigned long long>(), pool);
        else if (!any_mask && s->fast.ok)
            k_scan_fast<<<(int)g, SC_THREADS, 0, ctx->stream>>>(s->fast, cols, in->rows, O, s->cursor.as<unsigned long long>());
        else if (s->has_cond && (any_mask || s->has_div || s->has_null))
            k_scan_cond<true><<<(int)g, SC_THREADS, 0, ctx->stream>>>(reinterpret_cast<const ScanDev *>(s->dev.p), cols, in->rows, O,
                                                                      s->cursor.as<unsigned long long>(), s->flags.as<int32_t>(), pool, s->npool);
        else if (s->has_cond)
            k_scan_cond<false><<<(int)g, SC_THREADS, 0, ctx->stream>>>(reinterpret_cast<const ScanDev *>(s->dev.p), cols, in->rows, O,
                                                                       s->cursor.as<unsigned long long>(), s->flags.as<int32_t>(), pool, s->npool);
        else if (any_mask || s->has_div)
            k_scan<true><<<(int)g, SC_THREADS, 0, ctx->stream>>>(reinterpret_cast<const ScanDev *>(s->dev.p), cols, in->rows, O, s->cursor.as<unsigned long long>(),
                                                                 s->flags.as<int32_t>());
        else
            k_scan<false><<<(int)g, SC_THREADS, 0, ctx->stream>>>(reinterpret_cast<const ScanDev *>(s->dev.p), cols, in->rows, O, s->cursor.as<unsigned long long>(),
                                                                  s->flags.as<int32_t>());
    }
    GSQL_CUDA(ctx, cudaGetLastError());
    struct { unsigned long long n; unsigned long long pad; } h;
    int32_t hf[4];
    GSQL_CUDA(ctx, cudaMemcpyAsync(&h, s->cursor.p, 16, cudaMemcpyDeviceToHost, ctx->stream));
    GSQL_CUDA(ctx, cudaMemcpyAsync(hf, s->flags.p, 16, cudaMemcpyDeviceToHost, ctx->stream));
    GSQL_CUDA(ctx, cudaStreamSynchronize(ctx->stream));
    if (hf[0]) {
        cudaMemsetAsync(s->flags.p, 0, 16, ctx->stream);
        return gsql_set_error(ctx, GSQL_E_INVALID, "a NULL had to be written into an output column without a nulls buffer");
    }
    const int64_t n = (int64_t)h.n;
    GSQL_TRY(out_download(ctx, out, n, ob));
    *out_rows = out->rows = n;
    return GSQL_OK;
}
