// join.cu — GPU hash join behind gsql_join_* (drop-in for ParallelHashJoinExec build + probe).
//
// Reference path replaced (EX/ = polardbx-executor/src/main/java/com/alibaba/polardbx/executor/):
//   build : EX/operator/ParallelHashJoinExec.java:157-166 (consumeChunk), :107-128 (buildConsume), :388-426
//           (Synchronizer.initHashTable/buildHashTable), EX/utils/ExecUtils.java:914-944 (buildOneChunk),
//           EX/operator/util/ConcurrentRawHashTable.java:50-116
//   probe : EX/operator/AbstractBufferedJoinExec.java:185-264 (nextRows), AbstractHashJoinExec.java:80-106
//           (matchInit/matchNext), AbstractJoinExec.java:174-227 (row builders),
//           ParallelHashJoinExec.java:168-201,233-271 (outer-build variants)
//
// Layout (not the reference's): one open-addressing table of 16-byte slots {digest, chain head, multi flag}
// in HBM, two slots per 32-byte sector, load factor <= 0.5, slot = mulhi(fmix64(digest), nslots).  For a single
// key column the digest IS the key (exact, no verification read); for composite keys it is a 64-bit mix verified
// against the build columns.  Duplicate build keys hang off the slot as a LIFO chain through links[] exactly like
// positionLinks, and the `multi` flag lets the unique-key probe skip links[] entirely.
// Output is produced in two passes (count -> exclusive scan -> write) so it is dense and exactly sized.
#include <cub/device/device_scan.cuh>
#include <cub/iterator/transform_input_iterator.cuh>

#include "common.cuh"
#include "join_fast.cuh"

namespace {

constexpr unsigned long long DIGEST_EMPTY = 0x8000000000000000ULL;
enum { F_ANY_MULTI = 0, F_MORE_THAN_ONE = 1, F_NULL_INTO_NONNULL = 2, F_COUNT = 4 };
enum { SIDE_PROBE = 0, SIDE_BUILD = 1 };

struct __align__(16) Slot {
    unsigned long long digest;
    int head;
    int multi;
};

struct OutCol {
    void *data;
    uint8_t *nulls;
    int32_t type;
    int32_t side;
    int32_t col;
    int32_t pad;
};

struct ProbeParams {
    KeySet bkeys, pkeys;
    DColSet build, probe;
    const Slot *slots;
    const int32_t *links;
    uint8_t *used;  // build_outer: matched flags
    int32_t *flags;
    uint64_t nslots;
    int64_t probe_rows;
    int32_t join_type, single_join, semi_join, outer_join, build_outer, exact;
    int32_t n_anti;
    int32_t anti_cols[GSQL_MAX_KEYS];
    int32_t n_cond;
    int32_t cond_side[4], cond_col[4];
    int64_t cond_ne[4];
    int32_t nout;
    OutCol out[GSQL_MAX_COLS * 2];
};

// ------------------------------------------------------------------------------------------------ digests
// false => this row can never match (NULL key component, or NaN: Java `==` is false for NaN — DoubleBlock.java:77-91).
// A DOUBLE component is keyed by its bits, so -0.0 and +0.0 are different keys: the reference only pairs them when
// their hashes (0 and INT_MIN) happen to share a bucket, and the exchange, the bloom filter and the sort-merge join
// keep them apart too.
__device__ __forceinline__ bool key_digest(const KeySet &ks, int64_t r, unsigned long long &d) {
    if (ks.n == 1) {
        KeyVal k = gsql_load_key(ks.c[0], r, ks.utype[0]);
        if (k.is_null) return false;
        if (ks.utype[0] == GSQL_T_FP64 && __longlong_as_double(k.i) != __longlong_as_double(k.i)) return false;
        d = (unsigned long long)k.i;
        return true;
    }
    unsigned long long h = 0x243F6A8885A308D3ULL;
#pragma unroll 1
    for (int c = 0; c < ks.n; c++) {
        KeyVal k = gsql_load_key(ks.c[c], r, ks.utype[c]);
        if (k.is_null) return false;
        if (ks.utype[c] == GSQL_T_FP64 && __longlong_as_double(k.i) != __longlong_as_double(k.i)) return false;
        h = gsql_fmix64(h ^ (unsigned long long)k.i) + 0x9E3779B97F4A7C15ULL * (unsigned)(c + 1);
    }
    if (h == DIGEST_EMPTY) h ^= 1;
    d = h;
    return true;
}

__device__ __forceinline__ uint64_t slot_start(unsigned long long d, uint64_t nslots) {
    return __umul64hi(gsql_fmix64(d), nslots);
}

// Bit identity for every component (NaN components were never inserted / never probe, see key_digest).
__device__ __forceinline__ bool keys_equal(const KeySet &a, int64_t ra, const KeySet &b, int64_t rb) {
#pragma unroll 1
    for (int c = 0; c < a.n; c++) {
        KeyVal x = gsql_load_key(a.c[c], ra, a.utype[c]);
        KeyVal y = gsql_load_key(b.c[c], rb, b.utype[c]);
        if (x.is_null || y.is_null) return false;  // NULL components were never inserted / never probe
        if (x.i != y.i) return false;
    }
    return true;
}

// ------------------------------------------------------------------------------------------------ build
__global__ void __launch_bounds__(256) k_slots_init(Slot *slots, uint64_t n) {
    for (uint64_t i = blockIdx.x * (uint64_t)blockDim.x + threadIdx.x; i < n; i += (uint64_t)gridDim.x * blockDim.x) {
        int4 v;
        v.x = 0;
        v.y = (int)0x80000000;  // digest = 0x8000000000000000 (little endian: low word first)
        v.z = -1;               // head
        v.w = 0;                // multi
        reinterpret_cast<int4 *>(slots)[i] = v;
    }
}

__global__ void __launch_bounds__(256)
    k_join_build(KeySet bkeys, int64_t build_rows, Slot *slots, uint64_t nslots, int32_t *links, int32_t *flags) {
    for (int64_t p = blockIdx.x * (int64_t)blockDim.x + threadIdx.x; p < build_rows; p += (int64_t)gridDim.x * blockDim.x) {
        unsigned long long d;
        if (!key_digest(bkeys, p, d)) {  // ExecUtils.java:932-941: rows with a NULL key are never inserted
            links[p] = -1;
            continue;
        }
        uint64_t s;
        if (d == DIGEST_EMPTY) {
            s = nslots;  // dedicated slot for the one key that equals the empty marker
        } else {
            s = slot_start(d, nslots);
            while (true) {
                unsigned long long cur = *reinterpret_cast<volatile unsigned long long *>(&slots[s].digest);
                if (cur == DIGEST_EMPTY) {
                    unsigned long long prev = atomicCAS(&slots[s].digest, DIGEST_EMPTY, d);
                    if (prev == DIGEST_EMPTY || prev == d) break;
                } else if (cur == d) {
                    break;
                }
                if (++s == nslots) s = 0;
            }
        }
        int old = atomicExch(&slots[s].head, (int)p);  // newest row becomes the chain head (LIFO, like put())
        links[p] = old;
        if (old != -1) {
            slots[s].multi = 1;
            flags[F_ANY_MULTI] = 1;
        }
    }
}

// ------------------------------------------------------------------------------------------------ probe
__device__ __forceinline__ bool col_null(const DCol &c, int64_t r) { return c.nulls != nullptr && c.nulls[r] != 0; }

__device__ __forceinline__ int64_t col_int(const DCol &c, int64_t r) {
    if (c.type == GSQL_T_INT32) return reinterpret_cast<const int32_t *>(c.data)[r];
    if (c.type == GSQL_T_INT64) return reinterpret_cast<const int64_t *>(c.data)[r];
    return (int64_t) reinterpret_cast<const double *>(c.data)[r];
}

__device__ __forceinline__ void put_null(const ProbeParams &P, const OutCol &o, int64_t pos) {
    if (o.nulls) o.nulls[pos] = 1;
    else P.flags[F_NULL_INTO_NONNULL] = 1;
    if (o.type == GSQL_T_INT32) reinterpret_cast<int32_t *>(o.data)[pos] = 0;
    else reinterpret_cast<int64_t *>(o.data)[pos] = 0;
}

__device__ __forceinline__ void put_from(const ProbeParams &P, const OutCol &o, int64_t pos, const DCol &src, int64_t sr) {
    if (col_null(src, sr)) {
        put_null(P, o, pos);
        return;
    }
    if (o.nulls) o.nulls[pos] = 0;
    if (o.type == GSQL_T_INT32) reinterpret_cast<int32_t *>(o.data)[pos] = reinterpret_cast<const int32_t *>(src.data)[sr];
    else reinterpret_cast<int64_t *>(o.data)[pos] = reinterpret_cast<const int64_t *>(src.data)[sr];
}

// WRITE=false: returns the number of rows probe row r emits.  WRITE=true: writes them starting at `base`.
template <bool WRITE>
__device__ __forceinline__ int probe_one(const ProbeParams &P, int64_t r, int64_t base) {
    int emitted = 0;
    bool matched = false;
    unsigned long long d;
    if (key_digest(P.pkeys, r, d)) {
        // ---- find the slot of this digest (linear probing, stops at an empty slot)
        int head = -1, multi = 0;
        if (d == DIGEST_EMPTY) {
            Slot sl = P.slots[P.nslots];
            head = sl.head;
            multi = sl.multi;
        } else {
            uint64_t s = slot_start(d, P.nslots);
            while (true) {
                int4 raw = __ldg(reinterpret_cast<const int4 *>(&P.slots[s]));
                unsigned long long dg = ((unsigned long long)(unsigned)raw.y << 32) | (unsigned)raw.x;
                if (dg == d) {
                    head = raw.z;
                    multi = raw.w;
                    break;
                }
                if (dg == DIGEST_EMPTY) break;
                if (++s == P.nslots) s = 0;
            }
        }
        // ---- walk the chain (matchInit / matchNext)
        for (int m = head; m != -1; m = multi ? P.links[m] : -1) {
            if (!P.exact && !keys_equal(P.bkeys, m, P.pkeys, r)) continue;
            if (P.n_cond) {  // restricted otherCondition: joinRow[c] IS NULL OR joinRow[c] != v
                bool ok = true;
                for (int i = 0; i < P.n_cond && ok; i++) {
                    const DCol &c = P.cond_side[i] == SIDE_PROBE ? P.probe.c[P.cond_col[i]] : P.build.c[P.cond_col[i]];
                    int64_t row = P.cond_side[i] == SIDE_PROBE ? r : (int64_t)m;
                    if (!col_null(c, row) && col_int(c, row) == P.cond_ne[i]) ok = false;
                }
                if (!ok) continue;
            }
            if (!P.semi_join) {  // INNER / LEFT / RIGHT emit one joined row per match
                if (WRITE) {
                    int64_t pos = base + emitted;
                    for (int q = 0; q < P.nout; q++) {
                        const OutCol &o = P.out[q];
                        if (o.side == SIDE_PROBE) put_from(P, o, pos, P.probe.c[o.col], r);
                        else put_from(P, o, pos, P.build.c[o.col], m);
                    }
                    if (P.build_outer) P.used[m] = 1;  // markUsedKeys
                }
                emitted++;
            }
            if (P.single_join && matched) P.flags[F_MORE_THAN_ONE] = 1;  // AbstractBufferedJoinExec.java:217-219
            matched = true;
            if (P.semi_join) break;
        }
    }
    if (P.outer_join && !P.build_outer && !matched) {  // buildLeftNullRow / buildRightNullRow
        if (WRITE) {
            int64_t pos = base + emitted;
            for (int q = 0; q < P.nout; q++) {
                const OutCol &o = P.out[q];
                if (o.side == SIDE_PROBE) put_from(P, o, pos, P.probe.c[o.col], r);
                else put_null(P, o, pos);
            }
        }
        emitted++;
    }
    if (P.semi_join) {
        bool emit = false;
        if (P.join_type == GSQL_JOIN_SEMI) emit = matched;
        else if (!matched) {  // ANTI; checkAntiJoinOperands (AbstractJoinExec.java:126-136)
            emit = true;
            for (int i = 0; i < P.n_anti; i++)
                if (col_null(P.probe.c[P.anti_cols[i]], r)) emit = false;
        }
        if (emit) {
            if (WRITE) {
                int64_t pos = base + emitted;
                for (int q = 0; q < P.nout; q++) put_from(P, P.out[q], pos, P.probe.c[P.out[q].col], r);
            }
            emitted++;
        }
    }
    return emitted;
}

__global__ void __launch_bounds__(256) k_probe_count(const __grid_constant__ ProbeParams P, int32_t *__restrict__ cnt) {
    for (int64_t r = blockIdx.x * (int64_t)blockDim.x + threadIdx.x; r < P.probe_rows; r += (int64_t)gridDim.x * blockDim.x)
        cnt[r] = probe_one<false>(P, r, 0);
}

__global__ void __launch_bounds__(256) k_probe_write(const __grid_constant__ ProbeParams P, const int64_t *__restrict__ off) {
    for (int64_t r = blockIdx.x * (int64_t)blockDim.x + threadIdx.x; r < P.probe_rows; r += (int64_t)gridDim.x * blockDim.x)
        probe_one<true>(P, r, off[r]);
}

// unmatched build rows of an outer build (nextJoinNullRows)
__global__ void __launch_bounds__(256)
    k_unmatched_count(const uint8_t *__restrict__ used, int64_t rows, int32_t *__restrict__ cnt) {
    for (int64_t r = blockIdx.x * (int64_t)blockDim.x + threadIdx.x; r < rows; r += (int64_t)gridDim.x * blockDim.x)
        cnt[r] = used[r] ? 0 : 1;
}
__global__ void __launch_bounds__(256) k_unmatched_write(const __grid_constant__ ProbeParams P, int64_t build_rows,
                                                         const int64_t *__restrict__ off) {
    for (int64_t p = blockIdx.x * (int64_t)blockDim.x + threadIdx.x; p < build_rows; p += (int64_t)gridDim.x * blockDim.x) {
        if (P.used[p]) continue;
        int64_t pos = off[p];
        for (int q = 0; q < P.nout; q++) {
            const OutCol &o = P.out[q];
            if (o.side == SIDE_BUILD) put_from(P, o, pos, P.build.c[o.col], p);
            else put_null(P, o, pos);
        }
    }
}

struct ToI64 {
    __host__ __device__ int64_t operator()(const int32_t &v) const { return (int64_t)v; }
};

}  // namespace

// ================================================================================================ handle
struct gsql_join {
    gsql_ctx *ctx;
    gsql_join_spec spec;
    bool built = false;
    // build side
    int32_t n_build = 0, n_probe = 0;
    int32_t build_types[GSQL_MAX_COLS], probe_types[GSQL_MAX_COLS];
    int32_t bkey_cols[GSQL_MAX_KEYS], pkey_cols[GSQL_MAX_KEYS];
    RowStore store;
    bool aliased = false;  // gsql_join_build_consume_ref: the build columns are the caller's `alias`, not the store
    DColSet alias;
    int64_t build_rows = 0;
    // table
    DevBuf slots, links, used, flags;
    uint64_t nslots = 0;
    bool any_multi = false;
    bool generic_built = false;
    bool pass_nothing = false, pass_through = false;
    bool semi_join = false, outer_join = false, single_join = false;
    // output schema
    int32_t nout = 0;
    int32_t out_types[GSQL_MAX_COLS * 2];
    int32_t out_side[GSQL_MAX_COLS * 2], out_col[GSQL_MAX_COLS * 2];
    int32_t cond_side[4], cond_col[4];
    // fast path (join_fast.cuh)
    JoinFast fast;
};

extern "C" gsql_status gsql_join_create(gsql_ctx *ctx, const gsql_join_spec *spec, gsql_join **out) {
    if (!ctx || !spec || !out) return GSQL_E_INVALID;
    if (ctx->sticky) return GSQL_E_CUDA;
    *out = nullptr;
    const gsql_join_spec &s = *spec;
    if (s.join_type < GSQL_JOIN_INNER || s.join_type > GSQL_JOIN_ANTI) return gsql_set_error(ctx, GSQL_E_INVALID, "bad join type");
    if (s.nkeys < 1 || s.nkeys > GSQL_MAX_KEYS) return gsql_set_error(ctx, GSQL_E_INVALID, "need 1..%d equi keys", GSQL_MAX_KEYS);
    if (s.n_outer_cols < 1 || s.n_outer_cols > GSQL_MAX_COLS || s.n_inner_cols < 1 || s.n_inner_cols > GSQL_MAX_COLS)
        return gsql_set_error(ctx, GSQL_E_INVALID, "bad column counts");
    bool semi = (s.join_type == GSQL_JOIN_SEMI || s.join_type == GSQL_JOIN_ANTI) && !s.max_one_row;
    if ((s.join_type == GSQL_JOIN_SEMI || s.join_type == GSQL_JOIN_ANTI) && s.max_one_row)
        return gsql_set_error(ctx, GSQL_E_UNSUPPORTED, "single (max-one-row) semi/anti join");
    if (s.build_outer && (semi || s.n_cond > 0)) return gsql_set_error(ctx, GSQL_E_UNSUPPORTED, "build_outer with semi/anti/condition");
    if (s.n_cond < 0 || s.n_cond > 4 || s.n_anti_operands < 0 || s.n_anti_operands > GSQL_MAX_KEYS)
        return gsql_set_error(ctx, GSQL_E_INVALID, "bad condition / anti operand count");
    for (int i = 0; i < s.n_outer_cols; i++)
        if (s.outer_types[i] < GSQL_T_INT32 || s.outer_types[i] > GSQL_T_FP64) return gsql_set_error(ctx, GSQL_E_UNSUPPORTED, "outer col %d type", i);
    for (int i = 0; i < s.n_inner_cols; i++)
        if (s.inner_types[i] < GSQL_T_INT32 || s.inner_types[i] > GSQL_T_FP64) return gsql_set_error(ctx, GSQL_E_UNSUPPORTED, "inner col %d type", i);
    for (int i = 0; i < s.nkeys; i++) {
        if (s.outer_key[i] < 0 || s.outer_key[i] >= s.n_outer_cols || s.inner_key[i] < 0 || s.inner_key[i] >= s.n_inner_cols)
            return gsql_set_error(ctx, GSQL_E_INVALID, "key %d out of range", i);
        if (s.key_type[i] < GSQL_T_INT32 || s.key_type[i] > GSQL_T_FP64) return gsql_set_error(ctx, GSQL_E_INVALID, "key %d type", i);
    }
    for (int i = 0; i < s.n_anti_operands; i++)
        if (s.anti_operands[i] < 0 || s.anti_operands[i] >= s.n_outer_cols) return gsql_set_error(ctx, GSQL_E_INVALID, "anti operand");

    gsql_join *j = new gsql_join();
    j->ctx = ctx;
    gsql_ctx_retain(ctx);
    j->spec = s;
    j->semi_join = semi;
    j->single_join = s.max_one_row != 0;
    j->outer_join = s.join_type == GSQL_JOIN_LEFT || s.join_type == GSQL_JOIN_RIGHT;
    const bool bo = s.build_outer != 0;
    j->n_build = bo ? s.n_outer_cols : s.n_inner_cols;
    j->n_probe = bo ? s.n_inner_cols : s.n_outer_cols;
    for (int i = 0; i < j->n_build; i++) j->build_types[i] = bo ? s.outer_types[i] : s.inner_types[i];
    for (int i = 0; i < j->n_probe; i++) j->probe_types[i] = bo ? s.inner_types[i] : s.outer_types[i];
    for (int i = 0; i < s.nkeys; i++) {
        j->bkey_cols[i] = bo ? s.outer_key[i] : s.inner_key[i];
        j->pkey_cols[i] = bo ? s.inner_key[i] : s.outer_key[i];
    }
    j->store.init(j->build_types, j->n_build);
    // ---- output schema (AbstractJoinExec.java:103-120); outer -> probe unless build_outer
    const int outer_side = bo ? SIDE_BUILD : SIDE_PROBE, inner_side = bo ? SIDE_PROBE : SIDE_BUILD;
    auto push = [&](int side, int col, int type) {
        j->out_side[j->nout] = side;
        j->out_col[j->nout] = col;
        j->out_types[j->nout] = type;
        j->nout++;
    };
    if (semi) {
        for (int i = 0; i < s.n_outer_cols; i++) push(outer_side, i, s.outer_types[i]);
    } else if (j->single_join) {
        for (int i = 0; i < s.n_outer_cols; i++) push(outer_side, i, s.outer_types[i]);
        push(inner_side, 0, s.inner_types[0]);
    } else if (s.join_type == GSQL_JOIN_RIGHT) {
        for (int i = 0; i < s.n_inner_cols; i++) push(inner_side, i, s.inner_types[i]);
        for (int i = 0; i < s.n_outer_cols; i++) push(outer_side, i, s.outer_types[i]);
    } else {
        for (int i = 0; i < s.n_outer_cols; i++) push(outer_side, i, s.outer_types[i]);
        for (int i = 0; i < s.n_inner_cols; i++) push(inner_side, i, s.inner_types[i]);
    }
    // condition columns index the full join row leftSide || rightSide
    for (int i = 0; i < s.n_cond; i++) {
        int c = s.cond_col[i];
        int nleft = s.join_type == GSQL_JOIN_RIGHT ? s.n_inner_cols : s.n_outer_cols;
        int left_side = s.join_type == GSQL_JOIN_RIGHT ? inner_side : outer_side;
        int right_side = s.join_type == GSQL_JOIN_RIGHT ? outer_side : inner_side;
        if (c < 0 || c >= s.n_outer_cols + s.n_inner_cols) { delete j; gsql_ctx_release(ctx); return gsql_set_error(ctx, GSQL_E_INVALID, "cond col"); }
        j->cond_side[i] = c < nleft ? left_side : right_side;
        j->cond_col[i] = c < nleft ? c : c - nleft;
        int t = j->cond_side[i] == SIDE_PROBE ? j->probe_types[j->cond_col[i]] : j->build_types[j->cond_col[i]];
        if (t == GSQL_T_FP64) { delete j; gsql_ctx_release(ctx); return gsql_set_error(ctx, GSQL_E_UNSUPPORTED, "condition on a double column"); }
    }
    if (j->flags.alloc(ctx, F_COUNT * sizeof(int32_t)) != GSQL_OK) { delete j; gsql_ctx_release(ctx); return GSQL_E_OOM; }
    cudaMemsetAsync(j->flags.p, 0, j->flags.bytes, ctx->stream);
    *out = j;
    return GSQL_OK;
}

extern "C" void gsql_join_destroy(gsql_join *j) { destroy_handle(j); }

extern "C" gsql_status gsql_join_build_consume(gsql_join *j, const gsql_batch *b) {
    if (!j) return GSQL_E_INVALID;
    gsql_ctx *ctx = j->ctx;
    if (ctx->sticky) return GSQL_E_CUDA;
    if (j->built) return gsql_set_error(ctx, GSQL_E_STATE, "build_consume after build_finish");
    if (j->aliased) return gsql_set_error(ctx, GSQL_E_STATE, "build_consume after build_consume_ref");
    GSQL_TRY(validate_batch(ctx, b, j->n_build, j->build_types));
    if (b->rows == 0) return GSQL_OK;
    if (j->build_rows + b->rows > 0x7fffffffLL) return gsql_set_error(ctx, GSQL_E_UNSUPPORTED, "build side exceeds 2^31-1 rows");
    GSQL_CUDA(ctx, cudaSetDevice(ctx->device));
    GSQL_TRY(j->store.reserve(ctx, j->build_rows + b->rows, j->spec.expected_build_rows));
    GSQL_TRY(j->store.append(ctx, b, b->rows));
    if (b->mem == GSQL_MEM_HOST) GSQL_CUDA(ctx, cudaStreamSynchronize(ctx->stream));  // caller may reuse its buffers
    j->build_rows = j->store.rows;
    return GSQL_OK;
}

extern "C" gsql_status gsql_join_build_consume_ref(gsql_join *j, const gsql_batch *b) {
    if (!j) return GSQL_E_INVALID;
    gsql_ctx *ctx = j->ctx;
    if (ctx->sticky) return GSQL_E_CUDA;
    if (j->built) return gsql_set_error(ctx, GSQL_E_STATE, "build_consume_ref after build_finish");
    GSQL_TRY(validate_batch(ctx, b, j->n_build, j->build_types));
    if (b->mem != GSQL_MEM_DEVICE) return gsql_join_build_consume(j, b);  // host batches have to be uploaded anyway
    if (j->aliased || j->build_rows != 0) return gsql_set_error(ctx, GSQL_E_STATE, "build_consume_ref takes the whole build side as one batch");
    if (b->rows > 0x7fffffffLL) return gsql_set_error(ctx, GSQL_E_UNSUPPORTED, "build side exceeds 2^31-1 rows");
    if (b->rows == 0) return GSQL_OK;
    j->aliased = true;
    j->alias = batch_cols(b);
    j->build_rows = b->rows;
    return GSQL_OK;
}

static DColSet build_set(const gsql_join *j) { return j->aliased ? j->alias : j->store.view(); }

static void fill_build_cols(gsql_join *j, DColSet *build, KeySet *bkeys) {
    *build = build_set(j);
    bkeys->n = j->spec.nkeys;
    for (int i = 0; i < j->spec.nkeys; i++) {
        bkeys->c[i] = build->c[j->bkey_cols[i]];
        bkeys->utype[i] = j->spec.key_type[i];
    }
}


// ================================================================================================ fast path (host)
#define FJ_DISPATCH_W(W, ...)                              \
    switch (W) {                                           \
    case 1: { constexpr int WW = 1; __VA_ARGS__; } break;  \
    case 2: { constexpr int WW = 2; __VA_ARGS__; } break;  \
    case 3: { constexpr int WW = 3; __VA_ARGS__; } break;  \
    default: { constexpr int WW = 4; __VA_ARGS__; } break; \
    }

// The key-to-slot mode of the radix kernels (hash or direct table, join_fast.cuh KeyMap) as a compile-time DM.
#define FJ_DISPATCH_MODE(direct, ...)                   \
    if (direct) { constexpr bool DM = true; __VA_ARGS__; } \
    else { constexpr bool DM = false; __VA_ARGS__; }

// Rows per thread of the scatter k_fj_scatter_sm<W>: the most (<= sm_rpt_max(W)) whose tile fits one block's shared
// memory next to the kernel's static shared memory; 0 when not even one row per thread fits (fast_build then leaves
// the join to the generic path).
static gsql_status fj_scatter_rpt(gsql_ctx *ctx, int W, int P, int *rpt) {
    *rpt = 0;
    int optin = 0;
    GSQL_CUDA(ctx, cudaDeviceGetAttribute(&optin, cudaDevAttrMaxSharedMemoryPerBlockOptin, ctx->device));
    cudaFuncAttributes fa;
    FJ_DISPATCH_W(W, { GSQL_CUDA(ctx, cudaFuncGetAttributes(&fa, fj::k_fj_scatter_sm<WW, false>)); });  // static smem: same in both modes
    for (int r = fj::sm_rpt_max(W); r >= 1; r--)
        if (fj::scatter_sm_smem_bytes(W, P, r) + fa.sharedSizeBytes <= (size_t)optin) {
            *rpt = r;
            break;
        }
    return GSQL_OK;
}

// Block geometry shared by k_fj_hist and the scatter (offs is indexed [partition][block]): one block per SM and chunks
// of whole SM_THREADS * rpt-row tiles.
static fj::PartGeom fj_geom(gsql_ctx *ctx, int64_t rows, int P, int rpt) {
    fj::PartGeom g;
    g.rows = rows;
    g.P = P;
    const int64_t tile = (int64_t)fj::SM_THREADS * rpt;
    int64_t nblocks = ctx->sm_count;
    int64_t tiles = div_up(rows, tile);
    if (nblocks > tiles) nblocks = tiles;
    if (nblocks < 1) nblocks = 1;
    g.chunk = div_up(div_up(rows, nblocks), tile) * tile;
    g.nblocks = (int32_t)div_up(rows, g.chunk);
    if (g.nblocks < 1) g.nblocks = 1;
    return g;
}

// One-pass region layout for `rows` rows (RG->K == 0: use the exact layout).  A region holds its partition's mean share,
// two blocks per CTA (a partly filled current block and the reserved next one) and 8 sigma of binomial spread.  The
// probe reads every padding row, so the layout is taken only when the padding is at most 1/8 of the rows (C2: ~2.4 %).
// A block holds at least twice a tile's mean run per partition (and 256 rows), so a run rarely needs more than the next
// block; GSQL_JOIN_PART_BLOCK_ROWS sets K (rounded down to a power of two) for tests.
static gsql_status fj_region_plan(gsql_ctx *ctx, int64_t rows, int P, int W, fj::Regions *RG) {
    *RG = fj::Regions{};
    int rpt = 0;
    GSQL_TRY(fj_scatter_rpt(ctx, W, P, &rpt));
    if (P < 2 || rows < 1) return GSQL_OK;
    const fj::PartGeom g = fj_geom(ctx, rows, P, rpt);
    const int64_t T = (int64_t)fj::SM_THREADS * rpt;
    int64_t K = 256;
    while (K < 2 * T / P) K <<= 1;
    int64_t forced = 0;
    if (env_knob("GSQL_JOIN_PART_BLOCK_ROWS", &forced) && forced > 0)
        for (K = 1; K * 2 <= forced;) K <<= 1;
    const int64_t share = div_up(rows, P);
    const int64_t cap = div_up(share + 2 * K * g.nblocks + (int64_t)(8.0 * sqrt((double)share)) + K, K) * K;
    if ((cap * P - rows) * 8 > rows) return GSQL_OK;
    RG->cap = cap;
    RG->K = (int32_t)K;
    return GSQL_OK;
}

// Packs `rows` rows of `cols` into partition order.  Exact layout (RG.K == 0): out[rows * W] words, partitions back to
// back at offsets from a histogram pass and a scan.  Region layout (from fj_region_plan): one scatter pass fills
// out[P * RG.cap * W], region p = partition p, and every row no partition row took carries KEY_EMPTY; flags[FL_SPILL]
// reports a layout that could not be completed.  `direct`: partitions of the direct table.
static gsql_status fj_partition(gsql_ctx *ctx, const DColSet &cols, const fj::Layout &L, int64_t rows, int P, fj::Regions RG,
                                unsigned long long *out, int32_t *flags, const char *tag, bool direct, const fj::KeyMap &M) {
    const int W = L.nwords;
    int rpt = 0;
    GSQL_TRY(fj_scatter_rpt(ctx, W, P, &rpt));
    fj::PartGeom g = fj_geom(ctx, rows, P, rpt);
    if (RG.K) {
        DevBuf fill;
        GSQL_TRY(fill.alloc(ctx, (size_t)P * 8));
        GSQL_CUDA(ctx, cudaMemsetAsync(fill.p, 0, (size_t)P * 8, ctx->stream));
        RG.fill = fill.as<unsigned long long>();
        const size_t smem = fj::scatter_sm_smem_bytes(W, P, rpt);
        {
            KernelScope ks(ctx, (std::string("join_fast_scatter_") + tag).c_str());
            FJ_DISPATCH_W(W, FJ_DISPATCH_MODE(direct, {
                GSQL_CUDA(ctx, cudaFuncSetAttribute(fj::k_fj_scatter_sm<WW, DM>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));
                fj::k_fj_scatter_sm<WW, DM><<<g.nblocks, fj::SM_THREADS, smem, ctx->stream>>>(cols, L, g, rpt, nullptr, RG, out, flags, M);
            }));
        }
        GSQL_CUDA(ctx, cudaGetLastError());
        {
            KernelScope ks(ctx, (std::string("join_fast_gaps_") + tag).c_str());
            fj::k_fj_region_tail<<<P, 256, 0, ctx->stream>>>(RG, W, out);
        }
        GSQL_CUDA(ctx, cudaGetLastError());
        return GSQL_OK;
    }
    int64_t nh = (int64_t)P * g.nblocks;
    DevBuf hist, offs, tmp;
    GSQL_TRY(hist.alloc(ctx, (size_t)(nh + 1) * 8));
    GSQL_TRY(offs.alloc(ctx, (size_t)(nh + 1) * 8));
    GSQL_CUDA(ctx, cudaMemsetAsync((char *)hist.p + nh * 8, 0, 8, ctx->stream));
    std::string name = std::string("join_fast_hist_") + tag;
    {
        KernelScope ks(ctx, name.c_str());
        FJ_DISPATCH_MODE(direct, {
            fj::k_fj_hist<DM><<<g.nblocks, fj::SM_THREADS, (size_t)P * 4, ctx->stream>>>(cols.c[L.key_col], g, hist.as<int64_t>(), flags, M);
        });
    }
    GSQL_CUDA(ctx, cudaGetLastError());
    size_t tb = 0;
    GSQL_CUDA(ctx, cub::DeviceScan::ExclusiveSum(nullptr, tb, hist.as<int64_t>(), offs.as<int64_t>(), nh + 1, ctx->stream));
    GSQL_TRY(tmp.alloc(ctx, tb));
    name = std::string("join_fast_scan_") + tag;
    {
        KernelScope ks(ctx, name.c_str());
        GSQL_CUDA(ctx, cub::DeviceScan::ExclusiveSum(tmp.p, tb, hist.as<int64_t>(), offs.as<int64_t>(), nh + 1, ctx->stream));
    }
    const size_t smem = fj::scatter_sm_smem_bytes(W, P, rpt);
    name = std::string("join_fast_scatter_") + tag;
    {
        KernelScope ks(ctx, name.c_str());
        FJ_DISPATCH_W(W, FJ_DISPATCH_MODE(direct, {
            GSQL_CUDA(ctx, cudaFuncSetAttribute(fj::k_fj_scatter_sm<WW, DM>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));
            fj::k_fj_scatter_sm<WW, DM><<<g.nblocks, fj::SM_THREADS, smem, ctx->stream>>>(cols, L, g, rpt, offs.as<int64_t>(), RG, out, flags, M);
        }));
    }
    GSQL_CUDA(ctx, cudaGetLastError());
    return GSQL_OK;
}

// Builds the radix table from `packed` (build rows in partition order) one slot block at a time: k_fj_build_split groups
// the rows by block inside the table's own storage (a direct table's in a scratch area), k_fj_build_slab builds and writes every block (EMPTY slots included),
// k_fj_insert places the rows that either kernel deferred.  Blocks hold 2^lgB slots, the most whose slots fit 128 KB of shared
// memory (8192 for C2's W = 2; never fewer than MAX_DISP); GSQL_JOIN_BUILD_BLOCK_SLOTS overrides it (rounded down to
// a power of two, at least 2) so that tests can force tiny blocks.
static gsql_status fj_build_blocks(gsql_ctx *ctx, JoinFast &F, const unsigned long long *packed, int64_t rows, uint64_t spp) {
    const int W = F.bl.nwords;
    // shared-memory bits per slot: a whole row (hash), or the payload words and the occupancy bit (direct)
    const int64_t slot_bits = F.direct ? (int64_t)(W - 1) * 64 + 1 : (int64_t)W * 64;
    const int min_lgB = F.direct ? 5 : 1;  // direct: a block owns whole 32-bit bitmap words
    const int max_lgB = F.direct ? 16 : 62;  // direct, key-only rows: 8 KB of bitmap, 64 K rows per block
    int lgB = min_lgB;
    while (lgB < max_lgB && (2ll << lgB) * slot_bits / 8 <= (128ll << 10)) lgB++;
    int64_t forced = 0;
    if (env_knob("GSQL_JOIN_BUILD_BLOCK_SLOTS", &forced) && forced > 0) {
        int optin = 0;
        GSQL_CUDA(ctx, cudaDeviceGetAttribute(&optin, cudaDevAttrMaxSharedMemoryPerBlockOptin, ctx->device));
        lgB = min_lgB;
        while (lgB < max_lgB && (2ll << lgB) <= forced && (2ll << lgB) * slot_bits / 8 <= optin) lgB++;
    }
    const int64_t nb = (int64_t)((F.nslots + (1ull << lgB) - 1) >> lgB);
    // deferred rows: a few thousand for C2's hash table (~0.1 per block), none for a direct table unless a split CTA's
    // rows span more than its window of blocks; beyond the list the generic path takes over (FL_DISP)
    const int64_t def_cap = rows / 16 + 65536;
    DevBuf fill, def, ndef, scratch;
    GSQL_TRY(fill.alloc(ctx, (size_t)nb * 4));
    GSQL_TRY(def.alloc(ctx, (size_t)def_cap * W * 8));
    GSQL_TRY(ndef.alloc(ctx, 8));
    GSQL_CUDA(ctx, cudaMemsetAsync(fill.p, 0, fill.bytes, ctx->stream));
    GSQL_CUDA(ctx, cudaMemsetAsync(ndef.p, 0, 8, ctx->stream));
    unsigned long long *table = F.table.as<unsigned long long>();
    // where the split groups the rows by block: the hash table's own slots, or (direct table) a scratch area of whole rows
    unsigned long long *grouped = table;
    if (F.direct) {
        GSQL_TRY(scratch.alloc(ctx, (size_t)F.nslots * W * 8));
        grouped = scratch.as<unsigned long long>();
    }
    int32_t *flags = F.flags.as<int32_t>();
    FJ_DISPATCH_W(W, FJ_DISPATCH_MODE(F.direct, {
        {
            KernelScope ks(ctx, "join_fast_build_split");
            const size_t smem = fj::split_smem_bytes(WW);
            GSQL_CUDA(ctx, cudaFuncSetAttribute(fj::k_fj_build_split<WW, DM>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));
            int per_sm = 0;
            GSQL_CUDA(ctx, cudaOccupancyMaxActiveBlocksPerMultiprocessor(&per_sm, fj::k_fj_build_split<WW, DM>, fj::BS_THREADS, smem));
            if (per_sm < 1) per_sm = 1;
            const int64_t tile = (int64_t)fj::BS_THREADS * fj::bs_rpt(WW);
            int64_t grid = (int64_t)ctx->sm_count * per_sm;
            const int64_t tiles = div_up(rows, tile);
            if (grid > tiles) grid = tiles;
            const int64_t chunk = div_up(div_up(rows, grid), tile) * tile;
            grid = div_up(rows, chunk);
            fj::k_fj_build_split<WW, DM><<<(unsigned)grid, fj::BS_THREADS, smem, ctx->stream>>>(packed, rows, chunk, F.P, spp, F.nslots, lgB, grouped,
                                                                                             fill.as<unsigned int>(), def.as<unsigned long long>(),
                                                                                             ndef.as<unsigned long long>(), def_cap, flags, F.km);
        }
        GSQL_CUDA(ctx, cudaGetLastError());
        {
            KernelScope ks(ctx, "join_fast_build_slab");
            const size_t smem = (((size_t)1 << lgB) * slot_bits + 7) / 8;
            GSQL_CUDA(ctx, cudaFuncSetAttribute(fj::k_fj_build_slab<WW, DM>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));
            fj::k_fj_build_slab<WW, DM><<<(unsigned)nb, fj::BS_THREADS, smem, ctx->stream>>>(grouped, table, F.nslots, lgB, fill.as<unsigned int>(),
                                                                                            def.as<unsigned long long>(), ndef.as<unsigned long long>(),
                                                                                            def_cap, flags, F.km);
        }
        GSQL_CUDA(ctx, cudaGetLastError());
        {
            KernelScope ks(ctx, "join_fast_build_deferred");
            const int64_t tiles = div_up(def_cap, fj::TILE);
            const int grid = (int)(tiles < (int64_t)ctx->sm_count * 2 ? tiles : (int64_t)ctx->sm_count * 2);
            DColSet none;
            memset(&none, 0, sizeof(none));
            fj::k_fj_insert<WW, DM><<<grid, fj::THREADS, 0, ctx->stream>>>(def.as<unsigned long long>(), none, F.bl, def_cap, table, F.nslots, flags,
                                                                           ndef.as<unsigned long long>(), F.km);
        }
    }));
    GSQL_CUDA(ctx, cudaGetLastError());
    return GSQL_OK;
}

// Decides eligibility, builds the packed-row table; leaves j->fast.enabled = false when the generic path must run.
static gsql_status fast_build(gsql_join *j) {
    gsql_ctx *ctx = j->ctx;
    const gsql_join_spec &s = j->spec;
    JoinFast &F = j->fast;
    F.enabled = false;
    int64_t no_fast = 0;
    if (env_knob("GSQL_JOIN_NO_FAST", &no_fast) && no_fast) return GSQL_OK;
    if (s.nkeys != 1 || s.build_outer || j->single_join || s.n_cond > 0) return GSQL_OK;
    if (s.key_type[0] != GSQL_T_INT32 && s.key_type[0] != GSQL_T_INT64) return GSQL_OK;
    if (j->build_types[j->bkey_cols[0]] == GSQL_T_FP64 || j->probe_types[j->pkey_cols[0]] == GSQL_T_FP64) return GSQL_OK;
    if (s.key_type[0] == GSQL_T_INT32 && (j->build_types[j->bkey_cols[0]] != GSQL_T_INT32 || j->probe_types[j->pkey_cols[0]] != GSQL_T_INT32))
        return GSQL_OK;  // a BIGINT column narrowed to INT would not be the reference's conversion
    if (j->pass_nothing || j->pass_through || j->build_rows == 0) return GSQL_OK;
    const DColSet cols = build_set(j);
    for (int i = 0; i < j->n_build; i++)
        if (cols.c[i].nulls) return GSQL_OK;
    if (!fj::make_layout(j->build_types, j->n_build, j->bkey_cols[0], &F.bl)) return GSQL_OK;
    if (!fj::make_layout(j->probe_types, j->n_probe, j->pkey_cols[0], &F.pl)) return GSQL_OK;
    F.eligible = true;
    // A table that fits in L2 next to the streams (<= GSQL_JOIN_L2_TABLE_BYTES, 64 MB) is probed straight from the input
    // columns.  A larger one is radix-partitioned on the key hash into slices of GSQL_JOIN_PART_BYTES (16 MB): both
    // sides are packed into partition order, so every table access of the insert and of the probe hits a slice that
    // is resident in L2 — an unpartitioned probe pays a ~128-byte HBM fetch for each random 16-byte slot read
    const bool l2_table = !env_knob("GSQL_JOIN_PART_BYTES", &F.part_bytes);  // set, it forces the radix path (tests: small partitions)
    if (F.part_bytes < 4096) F.part_bytes = 4096;
    env_knob("GSQL_JOIN_SUB_BATCH", &F.sub_batch);
    if (F.sub_batch < fj::TILE) F.sub_batch = fj::TILE;
    env_knob("GSQL_JOIN_PART_MIN_ROWS", &F.part_min_rows);
    const int BW = F.bl.nwords;
    DColSet build;
    KeySet bkeys;
    fill_build_cols(j, &build, &bkeys);
    int64_t slots_per_row = 3;  // load factor 1/3: short probe sequences
    env_knob("GSQL_JOIN_SLOTS_PER_ROW", &slots_per_row);
    int64_t want = j->build_rows * slots_per_row;
    if (want < 1024) want = 1024;
    int64_t l2_bytes = 64ll << 20;
    env_knob("GSQL_JOIN_L2_TABLE_BYTES", &l2_bytes);
    int64_t P, spp;
    // The direct table when the build keys' range fits in 2^bits <= want slots: never more memory than the hash table,
    // one payload read per probe row (and a bitmap read unless the keys fill their range), and partitions of a
    // power-of-two slot count.  It stores no keys
    // ((W - 1) * 8 bytes and a bit per slot), but its partitions keep the slot ranges that W * 8-byte slots give
    // (spp * W * 8 <= part_bytes), so a partition's table slice is (W - 1) / W of part_bytes plus its bitmap.
    F.direct = false;
    {  // d_range is released before the table is allocated
        long long range[2] = {LLONG_MAX, LLONG_MIN};
        DevBuf d_range;
        GSQL_TRY(d_range.alloc(ctx, sizeof(range)));
        GSQL_CUDA(ctx, cudaMemcpyAsync(d_range.p, range, sizeof(range), cudaMemcpyHostToDevice, ctx->stream));
        {
            KernelScope ks(ctx, "join_key_range");
            fj::k_fj_key_range<<<grid_for(ctx, j->build_rows, 256, 8), 256, 0, ctx->stream>>>(build.c[F.bl.key_col], j->build_rows,
                                                                                                  d_range.as<long long>());
        }
        GSQL_CUDA(ctx, cudaGetLastError());
        GSQL_CUDA(ctx, cudaMemcpyAsync(range, d_range.p, sizeof(range), cudaMemcpyDeviceToHost, ctx->stream));
        GSQL_CUDA(ctx, cudaStreamSynchronize(ctx->stream));
        const uint64_t span = (uint64_t)range[1] - (uint64_t)range[0];
        int bits = 10;
        while (bits < 63 && (span >> bits) != 0) bits++;
        if (bits < 63 && (1ll << bits) <= want) {
            const int64_t nslots = 1ll << bits;
            spp = 1;
            while (spp < nslots && spp * 2 * BW * 8 <= F.part_bytes) spp *= 2;
            while (nslots / spp > fj::MAX_P) spp *= 2;
            if (l2_table && nslots * BW * 8 <= l2_bytes) spp = nslots;
            P = nslots / spp;
            F.direct = true;
            F.km.kmin = (unsigned long long)range[0];
            // as many rows as key values: with no duplicate (checked by the build) every value is a key
            F.km.dense = span + 1 == (uint64_t)j->build_rows ? span + 1 : 0;
            F.km.bits = bits;
            F.km.lgP = 0;
            while ((1ll << F.km.lgP) < P) F.km.lgP++;
        }
    }
    if (!F.direct) {
        P = div_up(want * BW * 8, F.part_bytes);
        if (l2_table && want * BW * 8 <= l2_bytes) P = 1;
        if (P > fj::MAX_P) P = fj::MAX_P;
        if (P < 1) P = 1;
        spp = div_up(want, P);
    }
    // the scatter must hold at least one row per thread of either side's packed rows at this P (always so on H100)
    int rb = 0, rp = 0;
    GSQL_TRY(fj_scatter_rpt(ctx, BW, (int)P, &rb));
    GSQL_TRY(fj_scatter_rpt(ctx, F.pl.nwords, (int)P, &rp));
    if (!rb || !rp) return GSQL_OK;
    F.P = (int)P;
    F.nslots = (uint64_t)(spp * P);
    GSQL_TRY(F.table.alloc(ctx, F.direct ? fj::direct_table_bytes(BW, F.nslots) : (size_t)F.nslots * BW * 8));
    GSQL_TRY(F.flags.alloc(ctx, fj::FL_COUNT * 4));
    GSQL_TRY(F.cursor.alloc(ctx, 8));
    GSQL_CUDA(ctx, cudaMemsetAsync(F.flags.p, 0, fj::FL_COUNT * 4, ctx->stream));
    DevBuf packed;
    // radix mode builds the table slot block by slot block; an unpartitioned table is EMPTY-filled and CAS-inserted
    const bool blocks = F.P > 1;
    if (!blocks) {
        KernelScope ks(ctx, "join_fast_table_init");
        if (F.direct) {  // an empty direct table is a clear bitmap (the payload words of unoccupied slots are never used)
            GSQL_CUDA(ctx, cudaMemsetAsync(F.table.as<unsigned long long>() + F.nslots * (BW - 1), 0, F.nslots / 8, ctx->stream));
        } else {
            int grid = grid_for(ctx, (int64_t)F.nslots, 256, 8);
            FJ_DISPATCH_W(BW, { fj::k_fj_table_init<WW><<<grid, 256, 0, ctx->stream>>>(F.table.as<unsigned long long>(), F.nslots); });
        }
    }
    const unsigned long long *src = nullptr;
    if (F.P > 1) {
        GSQL_TRY(packed.alloc(ctx, (size_t)j->build_rows * BW * 8));
        // exact layout: k_fj_build_split's chunk windows assume partitions back to back without gaps
        GSQL_TRY(fj_partition(ctx, build, F.bl, j->build_rows, F.P, fj::Regions{}, packed.as<unsigned long long>(), F.flags.as<int32_t>(), "build",
                              F.direct, F.km));
        src = packed.as<unsigned long long>();
    }
    if (blocks) {
        GSQL_TRY(fj_build_blocks(ctx, F, src, j->build_rows, (uint64_t)spp));
    } else {
        KernelScope ks(ctx, "join_fast_insert");
        int64_t itiles = div_up(j->build_rows, fj::TILE);
        int grid = (int)(itiles < (int64_t)ctx->sm_count * 2 ? itiles : (int64_t)ctx->sm_count * 2);
        FJ_DISPATCH_W(BW, FJ_DISPATCH_MODE(F.direct, {
            fj::k_fj_insert<WW, DM><<<grid, fj::THREADS, 0, ctx->stream>>>(src, build, F.bl, j->build_rows, F.table.as<unsigned long long>(), F.nslots,
                                                                           F.flags.as<int32_t>(), nullptr, F.km);
        }));
    }
    GSQL_CUDA(ctx, cudaGetLastError());
    int32_t hf[fj::FL_COUNT];
    GSQL_CUDA(ctx, cudaMemcpyAsync(hf, F.flags.p, sizeof(hf), cudaMemcpyDeviceToHost, ctx->stream));
    GSQL_CUDA(ctx, cudaStreamSynchronize(ctx->stream));
    if (hf[fj::FL_SENTINEL] || hf[fj::FL_DUP] || hf[fj::FL_DISP]) {  // not a unique-key table: generic chained path
        F.table.release();
        return GSQL_OK;
    }
    GSQL_CUDA(ctx, cudaMemsetAsync(F.flags.p, 0, fj::FL_COUNT * 4, ctx->stream));
    F.enabled = true;
    return GSQL_OK;
}


// Builds the generic chained table (lazily: the fast path only needs it for batches it cannot take).
static gsql_status ensure_generic(gsql_join *j) {
    if (j->generic_built) return GSQL_OK;
    gsql_ctx *ctx = j->ctx;
    const gsql_join_spec &s = j->spec;
    j->nslots = (uint64_t)(j->build_rows * 2 > 64 ? j->build_rows * 2 : 64);
    GSQL_TRY(j->slots.alloc(ctx, (size_t)(j->nslots + 1) * sizeof(Slot)));
    GSQL_TRY(j->links.alloc(ctx, (size_t)(j->build_rows > 0 ? j->build_rows : 1) * 4));
    if (s.build_outer) {
        GSQL_TRY(j->used.alloc(ctx, (size_t)(j->build_rows > 0 ? j->build_rows : 1)));
        GSQL_CUDA(ctx, cudaMemsetAsync(j->used.p, 0, j->used.bytes, ctx->stream));
    }
    {
        KernelScope ks(ctx, "join_slots_init");
        k_slots_init<<<grid_for(ctx, (int64_t)j->nslots + 1, 256, 8), 256, 0, ctx->stream>>>(j->slots.as<Slot>(), j->nslots + 1);
    }
    if (j->build_rows > 0) {
        DColSet build;
        KeySet bkeys;
        fill_build_cols(j, &build, &bkeys);
        KernelScope ks(ctx, "join_build");
        k_join_build<<<grid_for(ctx, j->build_rows, 256, 8), 256, 0, ctx->stream>>>(bkeys, j->build_rows, j->slots.as<Slot>(), j->nslots,
                                                                                        j->links.as<int32_t>(), j->flags.as<int32_t>());
    }
    GSQL_CUDA(ctx, cudaGetLastError());
    int32_t hflags[F_COUNT];
    GSQL_CUDA(ctx, cudaMemcpyAsync(hflags, j->flags.p, sizeof(hflags), cudaMemcpyDeviceToHost, ctx->stream));
    GSQL_CUDA(ctx, cudaStreamSynchronize(ctx->stream));
    j->any_multi = hflags[F_ANY_MULTI] != 0;
    j->generic_built = true;
    return GSQL_OK;
}

extern "C" gsql_status gsql_join_build_finish(gsql_join *j) {
    if (!j) return GSQL_E_INVALID;
    gsql_ctx *ctx = j->ctx;
    if (ctx->sticky) return GSQL_E_CUDA;
    if (j->built) return GSQL_OK;
    GSQL_CUDA(ctx, cudaSetDevice(ctx->device));
    const gsql_join_spec &s = j->spec;
    {  // a mask that never flagged a row is no mask: it must not cost the NULL-free fast path (a JNI caller hands over every Block's isNull[])
        const DColSet cols = build_set(j);
        const uint8_t *masks[GSQL_MAX_COLS];
        bool any[GSQL_MAX_COLS];
        for (int i = 0; i < j->n_build; i++) masks[i] = cols.c[i].nulls;
        GSQL_TRY(masks_any_null(ctx, j->n_build, masks, j->build_rows, GSQL_MEM_DEVICE, any));
        for (int i = 0; i < j->n_build; i++) {
            if (!masks[i] || any[i]) continue;
            if (j->aliased) j->alias.c[i].nulls = nullptr;
            else { j->store.has_nulls[i] = false; j->store.nulls[i].release(); }
        }
    }
    // pass-through / pass-nothing (ParallelHashJoinExec.buildConsume:107-128; doSpecialCheckForSemiJoin:290-310)
    if (j->build_rows == 0 && s.join_type == GSQL_JOIN_INNER) j->pass_nothing = true;
    if (j->semi_join) {
        if (j->build_rows == 0) {
            if (s.join_type == GSQL_JOIN_SEMI) j->pass_nothing = true;
            else j->pass_through = true;
        } else if (s.join_type == GSQL_JOIN_ANTI && s.n_anti_operands > 0 && j->n_build == 1 && build_set(j).c[0].nulls) {
            // x NOT IN (... NULL ...) is never true: need to know whether the single build column holds a NULL
            std::vector<uint8_t> h((size_t)j->build_rows);
            GSQL_CUDA(ctx, cudaMemcpyAsync(h.data(), build_set(j).c[0].nulls, (size_t)j->build_rows, cudaMemcpyDeviceToHost, ctx->stream));
            GSQL_CUDA(ctx, cudaStreamSynchronize(ctx->stream));
            for (uint8_t v : h)
                if (v) { j->pass_nothing = true; break; }
        }
    }
    GSQL_TRY(fast_build(j));
    if (!j->fast.enabled) GSQL_TRY(ensure_generic(j));
    j->built = true;
    return GSQL_OK;
}

extern "C" gsql_status gsql_join_info_get(gsql_join *j, gsql_join_info *info) {
    if (!j || !info) return GSQL_E_INVALID;
    memset(info, 0, sizeof(*info));
    info->build_rows = j->build_rows;
    info->table_slots = (int64_t)j->nslots;
    info->table_bytes = (int64_t)j->slots.bytes;
    info->device_bytes = (int64_t)(j->slots.bytes + j->links.bytes + j->used.bytes + j->store.bytes());
    info->has_duplicate_keys = j->any_multi;
    info->pass_through = j->pass_through;
    info->pass_nothing = j->pass_nothing;
    info->fast_path = j->fast.enabled ? 1 : 0;
    info->partitions = j->fast.enabled ? j->fast.P : 1;
    if (j->fast.enabled) { info->table_slots = (int64_t)j->fast.nslots; info->table_bytes = (int64_t)j->fast.table.bytes; info->device_bytes += (int64_t)j->fast.table.bytes; }
    return GSQL_OK;
}

extern "C" gsql_status gsql_join_output_schema(gsql_join *j, int32_t *ncols, int32_t *types) {
    if (!j || !ncols) return GSQL_E_INVALID;
    return output_schema(j->nout, j->out_types, ncols, types);
}

namespace {

// Everything a probe call holds in HBM besides the table.
struct ProbeWork {
    StagedBatch probe;
    DevBuf cnt, off, scan_tmp, total;
    OutBinding out;  // the probe's out batch, bound into ProbeParams::out by bind_out
};

gsql_status fill_params(gsql_join *j, const StagedBatch &sp, ProbeParams *P) {
    memset(P, 0, sizeof(*P));
    const gsql_join_spec &s = j->spec;
    fill_build_cols(j, &P->build, &P->bkeys);
    P->probe.n = sp.ncols;
    for (int i = 0; i < sp.ncols; i++) P->probe.c[i] = sp.cols[i];
    P->pkeys.n = s.nkeys;
    for (int i = 0; i < s.nkeys; i++) {
        P->pkeys.c[i] = sp.cols[j->pkey_cols[i]];
        P->pkeys.utype[i] = s.key_type[i];
    }
    P->slots = j->slots.as<Slot>();
    P->links = j->links.as<int32_t>();
    P->used = j->used.as<uint8_t>();
    P->flags = j->flags.as<int32_t>();
    P->nslots = j->nslots;
    P->probe_rows = sp.rows;
    P->join_type = s.join_type;
    P->single_join = j->single_join;
    P->semi_join = j->semi_join;
    P->outer_join = j->outer_join;
    P->build_outer = s.build_outer;
    P->exact = s.nkeys == 1;
    P->n_anti = s.n_anti_operands;
    for (int i = 0; i < s.n_anti_operands; i++) P->anti_cols[i] = s.anti_operands[i];
    P->n_cond = s.n_cond;
    for (int i = 0; i < s.n_cond; i++) {
        P->cond_side[i] = j->cond_side[i];
        P->cond_col[i] = j->cond_col[i];
        P->cond_ne[i] = s.cond_ne_value[i];
    }
    P->nout = j->nout;
    for (int q = 0; q < j->nout; q++) {
        P->out[q].type = j->out_types[q];
        P->out[q].side = j->out_side[q];
        P->out[q].col = j->out_col[q];
    }
    return GSQL_OK;
}

// count kernel + exclusive scan; leaves per-row offsets in w->off and returns the total.
gsql_status count_and_scan(gsql_join *j, const ProbeParams &P, int64_t rows, bool unmatched, ProbeWork *w, int64_t *total) {
    gsql_ctx *ctx = j->ctx;
    *total = 0;
    if (rows == 0) return GSQL_OK;
    GSQL_TRY(w->cnt.alloc(ctx, (size_t)rows * 4));
    GSQL_TRY(w->off.alloc(ctx, (size_t)(rows + 1) * 8));
    GSQL_TRY(w->total.alloc(ctx, 16));
    if (unmatched) {
        KernelScope ks(ctx, "join_unmatched_count");
        k_unmatched_count<<<grid_for(ctx, rows, 256, 8), 256, 0, ctx->stream>>>(j->used.as<uint8_t>(), rows, w->cnt.as<int32_t>());
    } else {
        KernelScope ks(ctx, "join_probe_count");
        k_probe_count<<<grid_for(ctx, rows, 256, 8), 256, 0, ctx->stream>>>(P, w->cnt.as<int32_t>());
    }
    GSQL_CUDA(ctx, cudaGetLastError());
    cub::TransformInputIterator<int64_t, ToI64, const int32_t *> in(w->cnt.as<int32_t>(), ToI64());
    size_t tmp = 0;
    GSQL_CUDA(ctx, cub::DeviceScan::ExclusiveSum(nullptr, tmp, in, w->off.as<int64_t>(), rows, ctx->stream));
    GSQL_TRY(w->scan_tmp.alloc(ctx, tmp));
    {
        KernelScope ks(ctx, "join_scan");
        GSQL_CUDA(ctx, cub::DeviceScan::ExclusiveSum(w->scan_tmp.p, tmp, in, w->off.as<int64_t>(), rows, ctx->stream));
    }
    int64_t last_off = 0;
    int32_t last_cnt = 0;
    GSQL_CUDA(ctx, cudaMemcpyAsync(&last_off, w->off.as<int64_t>() + (rows - 1), 8, cudaMemcpyDeviceToHost, ctx->stream));
    GSQL_CUDA(ctx, cudaMemcpyAsync(&last_cnt, w->cnt.as<int32_t>() + (rows - 1), 4, cudaMemcpyDeviceToHost, ctx->stream));
    GSQL_CUDA(ctx, cudaStreamSynchronize(ctx->stream));
    *total = last_off + last_cnt;
    return GSQL_OK;
}

gsql_status check_flags(gsql_join *j) {
    gsql_ctx *ctx = j->ctx;
    int32_t hflags[F_COUNT];
    GSQL_CUDA(ctx, cudaMemcpyAsync(hflags, j->flags.p, sizeof(hflags), cudaMemcpyDeviceToHost, ctx->stream));
    GSQL_CUDA(ctx, cudaStreamSynchronize(ctx->stream));
    if (hflags[F_MORE_THAN_ONE]) {
        int32_t zero = 0;
        cudaMemcpyAsync(j->flags.as<int32_t>() + F_MORE_THAN_ONE, &zero, 4, cudaMemcpyHostToDevice, ctx->stream);
        return gsql_set_error(ctx, GSQL_E_MORE_THAN_ONE_ROW, "ERR_SCALAR_SUBQUERY_RETURN_MORE_THAN_ONE_ROW");
    }
    if (hflags[F_NULL_INTO_NONNULL]) {
        int32_t zero = 0;
        cudaMemcpyAsync(j->flags.as<int32_t>() + F_NULL_INTO_NONNULL, &zero, 4, cudaMemcpyHostToDevice, ctx->stream);
        return gsql_set_error(ctx, GSQL_E_INVALID, "a NULL had to be written into an output column without a nulls buffer");
    }
    return GSQL_OK;
}

// Binds `rows` rows of `out` (out_bind) into P->out.
gsql_status bind_out(gsql_join *j, gsql_batch *out, int64_t rows, ProbeParams *P, ProbeWork *w) {
    GSQL_TRY(out_bind(j->ctx, out, rows, &w->out));
    for (int q = 0; q < j->nout; q++) {
        P->out[q].data = w->out.data[q];
        P->out[q].nulls = w->out.nulls[q];
    }
    return GSQL_OK;
}


static void fast_out_map(gsql_join *j, const ProbeParams &PP, fj::OutMap *O) {
    JoinFast &F = j->fast;
    memset(O, 0, sizeof(*O));
    O->nout = j->nout;
    O->join_type = j->spec.join_type;
    for (int q = 0; q < j->nout; q++) {
        const fj::Layout &L = j->out_side[q] == SIDE_PROBE ? F.pl : F.bl;
        O->data[q] = PP.out[q].data;
        O->nulls[q] = PP.out[q].nulls;
        O->side[q] = (int8_t)(j->out_side[q] == SIDE_PROBE ? 0 : 1);
        O->word[q] = (int8_t)L.word[j->out_col[q]];
        O->half[q] = (int8_t)L.half[j->out_col[q]];
        O->is32[q] = (int8_t)(j->out_types[q] == GSQL_T_INT32);
    }
}

// The region layout for a probe batch of m rows, or K == 0 for the exact one when the caller asks for it.
static gsql_status fj_probe_regions(gsql_join *j, int64_t m, bool exact, fj::Regions *RG) {
    JoinFast &F = j->fast;
    *RG = fj::Regions{};
    if (exact) return GSQL_OK;
    return fj_region_plan(j->ctx, m, F.P, F.pl.nwords, RG);
}

// Packed probe rows needed by batches of m1 and m2 rows (the full and the last sub-batch).
static gsql_status fj_probe_packed_rows(gsql_join *j, int64_t m1, int64_t m2, int64_t *rows) {
    *rows = m1 > m2 ? m1 : m2;
    for (int64_t m : {m1, m2}) {
        fj::Regions RG;
        GSQL_TRY(fj_probe_regions(j, m, false, &RG));
        if (RG.K && (int64_t)j->fast.P * RG.cap > *rows) *rows = (int64_t)j->fast.P * RG.cap;
    }
    return GSQL_OK;
}

// Partition (when P > 1) + probe of `m` device-resident rows; output rows are appended at *cursor.  Unless `exact`, the
// probe side may be partitioned in one pass into regions; if that layout spills, flags[FL_SPILL] is set, the probe
// emits nothing and the caller re-runs the batch with `exact`.
static gsql_status fast_probe_rows(gsql_join *j, const DColSet &cols, int64_t m, unsigned long long *packed, const fj::OutMap &O,
                                   unsigned long long *cursor, bool exact) {
    JoinFast &F = j->fast;
    gsql_ctx *ctx = j->ctx;
    const int PW = F.pl.nwords, BW = F.bl.nwords;
    const unsigned long long *src = nullptr;
    int64_t n = m;  // rows the probe walks: the padded length of a region layout
    fj::Regions RG{};
    // a batch too small to amortise the partitioning probes the (same) table directly
    if (F.P > 1 && m >= F.part_min_rows) {
        GSQL_TRY(fj_probe_regions(j, m, exact, &RG));
        GSQL_TRY(fj_partition(ctx, cols, F.pl, m, F.P, RG, packed, F.flags.as<int32_t>(), "probe", F.direct, F.km));
        if (RG.K) n = (int64_t)F.P * RG.cap;
        src = packed;
    }
    {
        KernelScope ks(ctx, "join_fast_probe");
        int grid = (int)div_up(n, fj::TILE);
        size_t smem = fj::stage_words_bytes(PW, BW, fj::TILE);
        const bool gaps = RG.K != 0;
#define FJ_PROBE_CASE(PWv, BWv)                                                                                                            \
    if (PW == PWv && BW == BWv) {                                                                                                          \
        FJ_DISPATCH_MODE(F.direct, {                                                                                                       \
            GSQL_CUDA(ctx, cudaFuncSetAttribute(fj::k_fj_probe<PWv, BWv, DM>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));    \
            fj::k_fj_probe<PWv, BWv, DM><<<grid, fj::THREADS, smem, ctx->stream>>>(src, cols, F.pl, n, gaps, F.table.as<unsigned long long>(), \
                                                                                  F.nslots, O, cursor, F.flags.as<int32_t>(), F.km);       \
        })                                                                                                                                 \
    }
        FJ_PROBE_CASE(1, 1) FJ_PROBE_CASE(1, 2) FJ_PROBE_CASE(1, 3) FJ_PROBE_CASE(1, 4)
        FJ_PROBE_CASE(2, 1) FJ_PROBE_CASE(2, 2) FJ_PROBE_CASE(2, 3) FJ_PROBE_CASE(2, 4)
        FJ_PROBE_CASE(3, 1) FJ_PROBE_CASE(3, 2) FJ_PROBE_CASE(3, 3) FJ_PROBE_CASE(3, 4)
        FJ_PROBE_CASE(4, 1) FJ_PROBE_CASE(4, 2) FJ_PROBE_CASE(4, 3) FJ_PROBE_CASE(4, 4)
#undef FJ_PROBE_CASE
    }
    GSQL_CUDA(ctx, cudaGetLastError());
    return GSQL_OK;
}

static bool fast_probe_applicable(gsql_join *j, const gsql_batch *probe, const gsql_batch *out, int64_t out_capacity, gsql_status *err) {
    *err = GSQL_OK;
    if (!j->fast.enabled) return false;
    if (out_capacity < probe->rows) return false;  // <= 1 output row per probe row; smaller buffers take the exact two-pass path
    for (int i = 0; i < probe->ncols; i++)
        if (probe->cols[i].nulls) return false;
    if (out->mem == GSQL_MEM_DEVICE)  // natural alignment of the caller's columns is enough (the flush aligns by address)
        for (int q = 0; q < j->nout; q++)
            if (((uintptr_t)out->cols[q].data & (uintptr_t)(gsql_type_width(j->out_types[q]) - 1)) != 0) return false;
    if (j->outer_join)
        for (int q = 0; q < j->nout; q++)
            if (j->out_side[q] == SIDE_BUILD && !out->cols[q].nulls) {
                *err = gsql_set_error(j->ctx, GSQL_E_INVALID, "outer join: output column %d needs a nulls buffer", q);
                return false;
            }
    return true;
}

// *spill: a one-pass probe layout spilled, so the call's output is incomplete and it must be re-run exactly (the flag
// is cleared).
static gsql_status fast_check_flags(gsql_join *j, bool *spill) {
    gsql_ctx *ctx = j->ctx;
    int32_t hf[fj::FL_COUNT];
    GSQL_CUDA(ctx, cudaMemcpyAsync(hf, j->fast.flags.p, sizeof(hf), cudaMemcpyDeviceToHost, ctx->stream));
    GSQL_CUDA(ctx, cudaStreamSynchronize(ctx->stream));
    if (hf[fj::FL_NULLOUT]) {
        cudaMemsetAsync(j->fast.flags.p, 0, fj::FL_COUNT * 4, ctx->stream);
        return gsql_set_error(ctx, GSQL_E_INVALID, "a NULL had to be written into an output column without a nulls buffer");
    }
    *spill = hf[fj::FL_SPILL] != 0;
    if (*spill) GSQL_CUDA(ctx, cudaMemsetAsync(j->fast.flags.as<int32_t>() + fj::FL_SPILL, 0, 4, ctx->stream));
    return GSQL_OK;
}

// Host batches: software pipeline over slices — H2D of slice i+1 (copy-in stream), partition+probe of slice i (compute
// stream) and D2H of slice i-1's output (copy-out stream) overlap, so the call is bound by max(PCIe in, PCIe out).
// *spill: see fast_check_flags.
static gsql_status fast_probe_host_pass(gsql_join *j, const gsql_batch *probe, gsql_batch *out, int64_t *out_rows, bool exact, bool *spill) {
    JoinFast &F = j->fast;
    gsql_ctx *ctx = j->ctx;
    const int64_t n = probe->rows;
    int64_t S = 16ll << 20;
    env_knob("GSQL_JOIN_HOST_SLICE", &S);
    if (S < fj::TILE) S = fj::TILE;
    if (S > n) S = n;
    const int nsl = (int)div_up(n, S);
    const int nc = probe->ncols, no = j->nout;
    const int PW = F.pl.nwords;
    int64_t packed_rows = 0;
    GSQL_TRY(fj_probe_packed_rows(j, S, n - (int64_t)(nsl - 1) * S, &packed_rows));
    std::vector<DevBuf> in((size_t)2 * nc), od((size_t)2 * no), on((size_t)2 * no);
    DevBuf packed, cursors;
    for (int b = 0; b < 2; b++) {
        for (int c = 0; c < nc; c++) GSQL_TRY(in[(size_t)b * nc + c].alloc(ctx, (size_t)S * gsql_type_width(j->probe_types[c])));
        for (int q = 0; q < no; q++) {
            GSQL_TRY(od[(size_t)b * no + q].alloc(ctx, (size_t)S * gsql_type_width(j->out_types[q])));
            if (out->cols[q].nulls) GSQL_TRY(on[(size_t)b * no + q].alloc(ctx, (size_t)S));
        }
    }
    if (F.P > 1) GSQL_TRY(packed.alloc(ctx, (size_t)packed_rows * PW * 8 + 64));
    GSQL_TRY(cursors.alloc(ctx, (size_t)nsl * 8));
    GSQL_CUDA(ctx, cudaMemsetAsync(cursors.p, 0, (size_t)nsl * 8, ctx->stream));
    unsigned long long *hcount = nullptr;
    GSQL_CUDA(ctx, cudaHostAlloc((void **)&hcount, (size_t)nsl * 8, cudaHostAllocDefault));
    std::vector<cudaEvent_t> in_done((size_t)nsl), comp_done((size_t)nsl), d2h_done((size_t)nsl);
    for (int i = 0; i < nsl; i++) {
        cudaEventCreateWithFlags(&in_done[(size_t)i], cudaEventDisableTiming);
        cudaEventCreateWithFlags(&comp_done[(size_t)i], cudaEventDisableTiming);
        cudaEventCreateWithFlags(&d2h_done[(size_t)i], cudaEventDisableTiming);
    }
    GSQL_CUDA(ctx, cudaStreamSynchronize(ctx->stream));  // buffers exist before the copy streams touch them
    gsql_status st = GSQL_OK;
    int64_t host_off = 0;
    auto drain = [&](int i) -> gsql_status {  // stage C for slice i
        GSQL_CUDA(ctx, cudaEventSynchronize(comp_done[(size_t)i]));
        int64_t cnt = (int64_t)hcount[i];
        int b = i & 1;
        for (int q = 0; q < no; q++) {
            size_t w = (size_t)gsql_type_width(j->out_types[q]);
            if (cnt > 0) {
                GSQL_CUDA(ctx, cudaMemcpyAsync((char *)out->cols[q].data + (size_t)host_off * w, od[(size_t)b * no + q].p, (size_t)cnt * w, cudaMemcpyDeviceToHost, ctx->copy_out));
                if (out->cols[q].nulls)
                    GSQL_CUDA(ctx, cudaMemcpyAsync(out->cols[q].nulls + host_off, on[(size_t)b * no + q].p, (size_t)cnt, cudaMemcpyDeviceToHost, ctx->copy_out));
            }
        }
        GSQL_CUDA(ctx, cudaEventRecord(d2h_done[(size_t)i], ctx->copy_out));
        host_off += cnt;
        return GSQL_OK;
    };
    for (int i = 0; i < nsl && st == GSQL_OK; i++) {
        const int b = i & 1;
        const int64_t lo = (int64_t)i * S, m = n - lo < S ? n - lo : S;
        // A: H2D of slice i (its buffer is free once slice i-2 has been computed)
        if (i >= 2) cudaStreamWaitEvent(ctx->copy_in, comp_done[(size_t)i - 2], 0);
        DColSet cols;
        memset(&cols, 0, sizeof(cols));
        cols.n = nc;
        for (int c = 0; c < nc && st == GSQL_OK; c++) {
            size_t w = (size_t)gsql_type_width(j->probe_types[c]);
            if (cudaMemcpyAsync(in[(size_t)b * nc + c].p, (const char *)probe->cols[c].data + (size_t)lo * w, (size_t)m * w, cudaMemcpyHostToDevice, ctx->copy_in) != cudaSuccess)
                st = gsql_set_error(ctx, GSQL_E_CUDA, "H2D slice copy failed");
            cols.c[c].data = in[(size_t)b * nc + c].p;
            cols.c[c].nulls = nullptr;
            cols.c[c].type = j->probe_types[c];
        }
        cudaEventRecord(in_done[(size_t)i], ctx->copy_in);
        // B: partition + probe of slice i
        cudaStreamWaitEvent(ctx->stream, in_done[(size_t)i], 0);
        if (i >= 2) cudaStreamWaitEvent(ctx->stream, d2h_done[(size_t)i - 2], 0);
        ProbeParams PP;
        memset(&PP, 0, sizeof(PP));
        for (int q = 0; q < no; q++) {
            PP.out[q].data = od[(size_t)b * no + q].p;
            PP.out[q].nulls = out->cols[q].nulls ? on[(size_t)b * no + q].as<uint8_t>() : nullptr;
        }
        fj::OutMap O;
        fast_out_map(j, PP, &O);
        if (st == GSQL_OK)
            st = fast_probe_rows(j, cols, m, packed.as<unsigned long long>(), O, cursors.as<unsigned long long>() + i, exact);
        cudaMemcpyAsync(&hcount[i], cursors.as<unsigned long long>() + i, 8, cudaMemcpyDeviceToHost, ctx->stream);
        cudaEventRecord(comp_done[(size_t)i], ctx->stream);
        // C: D2H of slice i-1's output
        if (i >= 1 && st == GSQL_OK) st = drain(i - 1);
    }
    if (st == GSQL_OK) st = drain(nsl - 1);
    cudaStreamSynchronize(ctx->copy_in);
    cudaStreamSynchronize(ctx->copy_out);
    cudaStreamSynchronize(ctx->stream);
    for (int i = 0; i < nsl; i++) {
        cudaEventDestroy(in_done[(size_t)i]);
        cudaEventDestroy(comp_done[(size_t)i]);
        cudaEventDestroy(d2h_done[(size_t)i]);
    }
    cudaFreeHost(hcount);
    if (st != GSQL_OK) return st;
    GSQL_TRY(fast_check_flags(j, spill));
    *out_rows = out->rows = host_off;
    return GSQL_OK;
}

static gsql_status fast_probe_host(gsql_join *j, const gsql_batch *probe, gsql_batch *out, int64_t *out_rows) {
    bool spill = false;
    GSQL_TRY(fast_probe_host_pass(j, probe, out, out_rows, false, &spill));
    if (spill) GSQL_TRY(fast_probe_host_pass(j, probe, out, out_rows, true, &spill));
    return GSQL_OK;
}

// Device-resident (or already staged) batch through the packed single-key table.
static gsql_status fast_probe(gsql_join *j, const StagedBatch &sp, gsql_batch *out, int64_t *out_rows) {
    JoinFast &F = j->fast;
    gsql_ctx *ctx = j->ctx;
    const int64_t n = sp.rows;
    ProbeWork w;
    ProbeParams PP;
    GSQL_TRY(fill_params(j, sp, &PP));
    GSQL_TRY(bind_out(j, out, n, &PP, &w));
    fj::OutMap O;
    fast_out_map(j, PP, &O);
    DColSet cols;
    memset(&cols, 0, sizeof(cols));
    cols.n = sp.ncols;
    DevBuf packed;
    const int64_t sub = F.P > 1 ? (F.sub_batch < n ? F.sub_batch : n) : n;
    if (F.P > 1) {
        int64_t packed_rows = 0;
        GSQL_TRY(fj_probe_packed_rows(j, sub, n - (div_up(n, sub) - 1) * sub, &packed_rows));
        GSQL_TRY(packed.alloc(ctx, (size_t)packed_rows * F.pl.nwords * 8 + 64));
    }
    unsigned long long total = 0;
    bool spill = false;
    for (int exact = 0; exact < 2; exact++) {  // a spilled one-pass layout: the whole call again, on the exact layout
        GSQL_CUDA(ctx, cudaMemsetAsync(F.cursor.p, 0, 8, ctx->stream));
        for (int64_t lo = 0; lo < n; lo += sub) {
            int64_t m = n - lo < sub ? n - lo : sub;
            for (int i = 0; i < sp.ncols; i++) {
                cols.c[i] = sp.cols[i];
                cols.c[i].data = (const char *)sp.cols[i].data + (size_t)lo * gsql_type_width(sp.cols[i].type);
            }
            GSQL_TRY(fast_probe_rows(j, cols, m, packed.as<unsigned long long>(), O, F.cursor.as<unsigned long long>(), exact != 0));
        }
        GSQL_CUDA(ctx, cudaMemcpyAsync(&total, F.cursor.p, 8, cudaMemcpyDeviceToHost, ctx->stream));
        GSQL_TRY(fast_check_flags(j, &spill));
        if (!spill) break;
    }
    GSQL_TRY(out_download(ctx, out, (int64_t)total, w.out));
    *out_rows = out->rows = (int64_t)total;
    return GSQL_OK;
}

}  // namespace

extern "C" gsql_status gsql_join_probe_count(gsql_join *j, const gsql_batch *probe, int64_t *out_rows) {
    if (!j || !out_rows) return GSQL_E_INVALID;
    gsql_ctx *ctx = j->ctx;
    if (ctx->sticky) return GSQL_E_CUDA;
    if (!j->built) return gsql_set_error(ctx, GSQL_E_STATE, "probe before build_finish");
    GSQL_TRY(validate_batch(ctx, probe, j->n_probe, j->probe_types));
    GSQL_CUDA(ctx, cudaSetDevice(ctx->device));
    *out_rows = 0;
    if (j->pass_nothing) return GSQL_OK;
    if (j->pass_through) { *out_rows = probe->rows; return GSQL_OK; }
    if (probe->rows == 0) return GSQL_OK;
    GSQL_TRY(ensure_generic(j));
    ProbeWork w;
    GSQL_TRY(stage_batch(ctx, probe, &w.probe));
    ProbeParams P;
    GSQL_TRY(fill_params(j, w.probe, &P));
    GSQL_TRY(count_and_scan(j, P, probe->rows, false, &w, out_rows));
    return check_flags(j);
}

extern "C" gsql_status gsql_join_probe(gsql_join *j, const gsql_batch *probe, gsql_batch *out, int64_t out_capacity, int64_t *out_rows) {
    if (!j || !out || !out_rows) return GSQL_E_INVALID;
    gsql_ctx *ctx = j->ctx;
    if (ctx->sticky) return GSQL_E_CUDA;
    if (!j->built) return gsql_set_error(ctx, GSQL_E_STATE, "probe before build_finish");
    GSQL_TRY(validate_batch(ctx, probe, j->n_probe, j->probe_types));
    GSQL_TRY(validate_batch(ctx, out, j->nout, j->out_types));
    if (out->mem != probe->mem) return gsql_set_error(ctx, GSQL_E_INVALID, "probe and out must live in the same memory space");
    GSQL_CUDA(ctx, cudaSetDevice(ctx->device));
    *out_rows = 0;
    out->rows = 0;
    if (j->pass_nothing || probe->rows == 0) return GSQL_OK;
    if (j->pass_through) {  // ANTI with an empty build side: every probe row passes (even NULL operands)
        if (out_capacity < probe->rows) { *out_rows = probe->rows; return gsql_set_error(ctx, GSQL_E_CAPACITY, "need %lld rows", (long long)probe->rows); }
        cudaMemcpyKind kind = probe->mem == GSQL_MEM_DEVICE ? cudaMemcpyDeviceToDevice : cudaMemcpyHostToHost;
        for (int q = 0; q < j->nout; q++) {
            const gsql_col &src = probe->cols[j->out_col[q]];
            GSQL_CUDA(ctx, cudaMemcpyAsync(out->cols[q].data, src.data, (size_t)probe->rows * gsql_type_width(src.type), kind, ctx->stream));
            if (src.nulls) {
                if (!out->cols[q].nulls) return gsql_set_error(ctx, GSQL_E_INVALID, "output column %d needs a nulls buffer", q);
                GSQL_CUDA(ctx, cudaMemcpyAsync(out->cols[q].nulls, src.nulls, (size_t)probe->rows, kind, ctx->stream));
            } else if (out->cols[q].nulls) {
                if (probe->mem == GSQL_MEM_DEVICE) GSQL_CUDA(ctx, cudaMemsetAsync(out->cols[q].nulls, 0, (size_t)probe->rows, ctx->stream));
                else memset(out->cols[q].nulls, 0, (size_t)probe->rows);
            }
        }
        GSQL_CUDA(ctx, cudaStreamSynchronize(ctx->stream));
        *out_rows = out->rows = probe->rows;
        return GSQL_OK;
    }
    ProbeWork w;
    gsql_batch stripped;
    gsql_col stripped_cols[GSQL_MAX_COLS];
    if (j->fast.enabled) {  // all-zero null masks are dropped before the path is chosen
        bool has_mask = false;
        for (int i = 0; i < probe->ncols; i++) has_mask |= probe->cols[i].nulls != nullptr;
        if (has_mask) {
            GSQL_TRY(strip_zero_masks(ctx, probe, &stripped, stripped_cols));
            probe = &stripped;
        }
    }
    {
        gsql_status ferr = GSQL_OK;
        bool fast = fast_probe_applicable(j, probe, out, out_capacity, &ferr);
        if (ferr != GSQL_OK) return ferr;
        if (fast && probe->mem == GSQL_MEM_HOST && probe->rows >= (1 << 20)) return fast_probe_host(j, probe, out, out_rows);
        GSQL_TRY(stage_batch(ctx, probe, &w.probe));
        if (fast) return fast_probe(j, w.probe, out, out_rows);
    }
    GSQL_TRY(ensure_generic(j));
    ProbeParams P;
    GSQL_TRY(fill_params(j, w.probe, &P));
    int64_t total = 0;
    GSQL_TRY(count_and_scan(j, P, probe->rows, false, &w, &total));
    GSQL_TRY(check_flags(j));
    if (total > out_capacity) {
        *out_rows = total;
        return gsql_set_error(ctx, GSQL_E_CAPACITY, "output needs %lld rows, capacity %lld", (long long)total, (long long)out_capacity);
    }
    if (total > 0) {
        GSQL_TRY(bind_out(j, out, total, &P, &w));
        {
            KernelScope ks(ctx, "join_probe_write");
            k_probe_write<<<grid_for(ctx, probe->rows, 256, 8), 256, 0, ctx->stream>>>(P, w.off.as<int64_t>());
        }
        GSQL_CUDA(ctx, cudaGetLastError());
        GSQL_TRY(check_flags(j));
        GSQL_TRY(out_download(ctx, out, total, w.out));
    }
    *out_rows = out->rows = total;
    return GSQL_OK;
}

extern "C" gsql_status gsql_join_unmatched_build(gsql_join *j, gsql_batch *out, int64_t out_capacity, int64_t *out_rows) {
    if (!j || !out || !out_rows) return GSQL_E_INVALID;
    gsql_ctx *ctx = j->ctx;
    if (ctx->sticky) return GSQL_E_CUDA;
    if (!j->built) return gsql_set_error(ctx, GSQL_E_STATE, "unmatched_build before build_finish");
    GSQL_TRY(validate_batch(ctx, out, j->nout, j->out_types));
    *out_rows = 0;
    out->rows = 0;
    if (!j->spec.build_outer || !j->outer_join || j->build_rows == 0) return GSQL_OK;
    GSQL_CUDA(ctx, cudaSetDevice(ctx->device));
    GSQL_TRY(ensure_generic(j));
    ProbeWork w;
    w.probe.rows = 0;
    w.probe.ncols = j->n_probe;
    for (int i = 0; i < j->n_probe; i++) w.probe.cols[i] = DCol{nullptr, nullptr, j->probe_types[i], 0};
    ProbeParams P;
    GSQL_TRY(fill_params(j, w.probe, &P));
    int64_t total = 0;
    GSQL_TRY(count_and_scan(j, P, j->build_rows, true, &w, &total));
    if (total > out_capacity) {
        *out_rows = total;
        return gsql_set_error(ctx, GSQL_E_CAPACITY, "output needs %lld rows, capacity %lld", (long long)total, (long long)out_capacity);
    }
    if (total > 0) {
        GSQL_TRY(bind_out(j, out, total, &P, &w));
        {
            KernelScope ks(ctx, "join_unmatched_write");
            k_unmatched_write<<<grid_for(ctx, j->build_rows, 256, 8), 256, 0, ctx->stream>>>(P, j->build_rows, w.off.as<int64_t>());
        }
        GSQL_CUDA(ctx, cudaGetLastError());
        GSQL_TRY(check_flags(j));
        GSQL_TRY(out_download(ctx, out, total, w.out));
    }
    *out_rows = out->rows = total;
    return GSQL_OK;
}
