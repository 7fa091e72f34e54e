// common.cuh — shared host/device pieces of libgsql_gpu.so (sm_90a only).
//
// Hash restatements are bit-exact with the reference (file:line cited at each function) because they are
// observable across the exchange boundary (a GPU task and a stock Java task must route a row to the same
// consumer).  The join / group-by tables themselves are NOT the reference's structures: only the result
// multiset is contractual (BaseExecTest.java:78-103), so they are laid out for HBM sectors instead.
#pragma once

#include <cuda_runtime.h>
#include <stdint.h>
#include <stdio.h>
#include <string.h>

#include <string>
#include <vector>

#include "../../include/gsql_gpu.h"

// ------------------------------------------------------------------------------------------------ context
struct ProfEntry {
    std::string name;
    int64_t launches = 0;
    double ms = 0;
    std::vector<std::pair<cudaEvent_t, cudaEvent_t>> pending;
};

struct gsql_ctx {
    int device = 0;
    cudaStream_t stream = nullptr;
    bool own_stream = false;
    cudaStream_t copy_in = nullptr;   // H2D staging stream (e2e path)
    cudaStream_t copy_out = nullptr;  // D2H staging stream
    char err[1024] = {0};
    bool sticky = false;
    bool profiling = false;
    std::vector<ProfEntry> prof;
    std::vector<cudaEvent_t> event_pool;
    int64_t launches = 0;
    void *nccl_comm = nullptr;  // ncclComm_t
    // extra communicators (ncclCommSplit) + streams: the AllToAllv is striped over them so that several NCCL p2p
    // kernels move data concurrently (one communicator alone stays far below the NVLink rate)
    void *nccl_extra[7] = {nullptr, nullptr, nullptr, nullptr, nullptr, nullptr, nullptr};
    cudaStream_t xstreams[7] = {nullptr, nullptr, nullptr, nullptr, nullptr, nullptr, nullptr};
    int n_extra = 0;
    int nranks = 1, rank = 0;
    int sm_count = 132;
    int refs = 1;  // the creator + every live handle: a handle may be destroyed after gsql_ctx_destroy (GC order)
};

void gsql_ctx_retain(gsql_ctx *ctx);
void gsql_ctx_release(gsql_ctx *ctx);

gsql_status gsql_set_error(gsql_ctx *ctx, gsql_status st, const char *fmt, ...);

#define GSQL_CUDA(ctx, call)                                                                                   \
    do {                                                                                                       \
        cudaError_t _e = (call);                                                                               \
        if (_e != cudaSuccess) {                                                                               \
            (ctx)->sticky = true;                                                                              \
            return gsql_set_error((ctx), _e == cudaErrorMemoryAllocation ? GSQL_E_OOM : GSQL_E_CUDA,           \
                                  "%s:%d %s -> %s", __FILE__, __LINE__, #call, cudaGetErrorString(_e));        \
        }                                                                                                      \
    } while (0)

#define GSQL_TRY(expr)                    \
    do {                                  \
        gsql_status _s = (expr);          \
        if (_s != GSQL_OK) return _s;     \
    } while (0)

// RAII scope that times one named kernel launch with CUDA events on the launching stream (profiling only) and
// counts the launch.  Usage:  { KernelScope ks(ctx, "join_probe"); kernel<<<g, b, 0, ctx->stream>>>(...); }
struct KernelScope {
    gsql_ctx *ctx;
    int idx = -1;
    cudaEvent_t start = nullptr;
    cudaStream_t stream = nullptr;  // the stream the kernel is launched on (default: the context stream)
    KernelScope(gsql_ctx *c, const char *name, cudaStream_t on = nullptr);
    ~KernelScope();
};

// Stream-ordered device memory (cudaMallocAsync on the context stream).
gsql_status dev_alloc(gsql_ctx *ctx, size_t bytes, void **out);
void dev_free(gsql_ctx *ctx, void *p);

struct DevBuf {
    gsql_ctx *ctx = nullptr;
    void *p = nullptr;
    size_t bytes = 0;
    DevBuf() {}
    DevBuf(const DevBuf &) = delete;
    DevBuf &operator=(const DevBuf &) = delete;
    ~DevBuf() { release(); }
    void release() {
        if (p && ctx) dev_free(ctx, p);
        p = nullptr;
        bytes = 0;
    }
    gsql_status alloc(gsql_ctx *c, size_t n) {
        release();
        ctx = c;
        if (n == 0) n = 16;
        gsql_status s = dev_alloc(c, n, &p);
        if (s == GSQL_OK) bytes = n;
        return s;
    }
    // Grow keeping the first `keep` bytes.
    gsql_status grow(gsql_ctx *c, size_t n, size_t keep) {
        if (n <= bytes) return GSQL_OK;
        void *np = nullptr;
        gsql_status s = dev_alloc(c, n, &np);
        if (s != GSQL_OK) return s;
        if (p && keep) {
            cudaError_t e = cudaMemcpyAsync(np, p, keep, cudaMemcpyDeviceToDevice, c->stream);
            if (e != cudaSuccess) return gsql_set_error(c, GSQL_E_CUDA, "grow copy: %s", cudaGetErrorString(e));
        }
        if (p) dev_free(c, p);
        ctx = c;
        p = np;
        bytes = n;
        return GSQL_OK;
    }
    template <typename T> T *as() const { return reinterpret_cast<T *>(p); }
};

// ------------------------------------------------------------------------------------------------ columns
__host__ __device__ inline int gsql_type_width(int t) { return t == GSQL_T_INT32 ? 4 : (t == GSQL_T_DEC128 ? 16 : 8); }

struct DCol {  // a Block resident in HBM
    const void *data;
    const uint8_t *nulls;  // nullptr = no NULLs
    int32_t type;
    int32_t pad;
};

struct DColSet {
    int32_t n;
    int32_t pad;
    DCol c[GSQL_MAX_COLS];
};

struct KeySet {  // key columns with their unified type (EquiJoinKey.unifiedType / keyTargetTypes)
    int32_t n;
    int32_t pad;
    DCol c[GSQL_MAX_KEYS];
    int32_t utype[GSQL_MAX_KEYS];
};

// A batch staged in HBM: aliases device input or owns uploaded copies of host input.
struct StagedBatch {
    int64_t rows = 0;
    int32_t ncols = 0;
    DCol cols[GSQL_MAX_COLS];
    std::vector<DevBuf *> owned;
    ~StagedBatch() {
        for (auto *b : owned) delete b;
    }
};
gsql_status stage_batch(gsql_ctx *ctx, const gsql_batch *in, StagedBatch *out);
gsql_status validate_batch(gsql_ctx *ctx, const gsql_batch *b, int32_t expect_cols, const int32_t *expect_types);
// any[i] = mask i holds a non-zero byte (masks[i] == nullptr -> false).  One kernel + one 4*n-byte read-back for device
// masks, a word-wise host scan for host masks.  A Block that carries an all-zero boolean[] isNull (the reference allows
// it: AbstractBlock.mayHaveNull() is only a hint) must not cost the NULL-free fast paths.
gsql_status masks_any_null(gsql_ctx *ctx, int n, const uint8_t *const *masks, int64_t rows, int mem, bool *any);
// Copy of `in` whose all-zero null masks are dropped (cols_storage: GSQL_MAX_COLS entries owned by the caller).
gsql_status strip_zero_masks(gsql_ctx *ctx, const gsql_batch *in, gsql_batch *out, gsql_col *cols_storage);

// ------------------------------------------------------------------------------------------------ hashing
// fastutil HashCommon.mix (call sites ConcurrentRawHashTable.java:93,114; GroupOpenHashMap.java:143)
__host__ __device__ __forceinline__ int32_t gsql_mix(int32_t x) {
    uint32_t h = (uint32_t)x * 0x9E3779B9u;
    return (int32_t)(h ^ (h >> 16));
}
// fastutil HashCommon.murmurHash3 (call site ExecUtils.java:1026,1029)
__host__ __device__ __forceinline__ int32_t gsql_murmur3(int32_t xi) {
    uint32_t x = (uint32_t)xi;
    x ^= x >> 16;
    x *= 0x85ebca6bu;
    x ^= x >> 13;
    x *= 0xc2b2ae35u;
    x ^= x >> 16;
    return (int32_t)x;
}
// ExecUtils.partition (EX/utils/ExecUtils.java:1023-1031)
__host__ __device__ __forceinline__ int32_t gsql_partition_of(int32_t hash, int32_t nparts, bool pow2) {
    uint32_t m = (uint32_t)gsql_murmur3(hash);
    return pow2 ? (int32_t)(m & (uint32_t)(nparts - 1)) : (int32_t)((m & 0x7fffffffu) % (uint32_t)nparts);
}
// Long.hashCode (LongBlock.java:110-115)
__host__ __device__ __forceinline__ int32_t gsql_hash_i64(int64_t v) {
    uint64_t u = (uint64_t)v;
    return (int32_t)(uint32_t)(u ^ (u >> 32));
}
// Double.doubleToLongBits: NaN canonicalised (DoubleBlock.java:111-116)
__device__ __forceinline__ int64_t gsql_double_bits(double d) {
    return d != d ? 0x7ff8000000000000LL : __double_as_longlong(d);
}

struct KeyVal {
    int64_t i;  // integer value, or raw double bits for FP64
    bool is_null;
};

// Reads key column c at row r converted to its unified type (Converters.java:94-131): integer widening or
// (double) cast.  For FP64 the value travels as raw (non-canonicalised) bits.
__device__ __forceinline__ KeyVal gsql_load_key(const DCol &c, int64_t r, int utype) {
    KeyVal k;
    k.is_null = c.nulls != nullptr && c.nulls[r] != 0;
    k.i = 0;
    if (k.is_null) return k;
    // input columns are read once: evict-first loads keep the L2 for the hash-table slices (see ld_stream_* below)
    if (utype == GSQL_T_FP64) {
        double d;
        if (c.type == GSQL_T_FP64) d = __ldcs(reinterpret_cast<const double *>(c.data) + r);
        else if (c.type == GSQL_T_INT64) d = (double)__ldcs(reinterpret_cast<const long long *>(c.data) + r);
        else d = (double)__ldcs(reinterpret_cast<const int *>(c.data) + r);
        k.i = __double_as_longlong(d);
    } else {
        if (c.type == GSQL_T_INT32) k.i = __ldcs(reinterpret_cast<const int *>(c.data) + r);
        else if (c.type == GSQL_T_INT64) k.i = __ldcs(reinterpret_cast<const long long *>(c.data) + r);
        else k.i = (int64_t)__ldcs(reinterpret_cast<const double *>(c.data) + r);
    }
    return k;
}
// Block.hashCode(position) per unified type; NULL -> 0 (Block.java:113-118, IntegerBlock.java:112-117)
__device__ __forceinline__ int32_t gsql_key_hash(const KeyVal &k, int utype) {
    if (k.is_null) return 0;
    if (utype == GSQL_T_INT32) return (int32_t)k.i;
    if (utype == GSQL_T_FP64) return gsql_hash_i64(gsql_double_bits(__longlong_as_double(k.i)));
    return gsql_hash_i64(k.i);
}
// Chunk.hashCode(position): h = h*31 + block.hashCode (Chunk.java:124-130)
__device__ __forceinline__ int32_t gsql_row_hash(const KeySet &ks, int64_t r) {
    uint32_t h = 0;
#pragma unroll 1
    for (int c = 0; c < ks.n; c++) {
        KeyVal k = gsql_load_key(ks.c[c], r, ks.utype[c]);
        h = h * 31u + (uint32_t)gsql_key_hash(k, ks.utype[c]);
    }
    return (int32_t)h;
}

// 64-bit finaliser used for table placement (not contractual).
__host__ __device__ __forceinline__ uint64_t gsql_fmix64(uint64_t x) {
    x ^= x >> 33;
    x *= 0xff51afd7ed558ccdULL;
    x ^= x >> 33;
    x *= 0xc4ceb9fe1a85ec53ULL;
    x ^= x >> 33;
    return x;
}

// ------------------------------------------------------------------------------------------------ memory ops
// Streaming (read-once) loads / write-once stores use the .cs (evict-first) policy so that hash-table sectors stay
// resident in the L2 (50 MB on H100); table reads carry an explicit L2 evict_last cache policy.
__device__ __forceinline__ int4 ld_stream_16(const void *p) { return __ldcs(reinterpret_cast<const int4 *>(p)); }
__device__ __forceinline__ long long ld_stream_8(const void *p) { return __ldcs(reinterpret_cast<const long long *>(p)); }
__device__ __forceinline__ int ld_stream_4(const void *p) { return __ldcs(reinterpret_cast<const int *>(p)); }
__device__ __forceinline__ void st_stream_16(void *p, const int4 &v) { __stcs(reinterpret_cast<int4 *>(p), v); }
__device__ __forceinline__ void st_stream_8(void *p, long long v) { __stcs(reinterpret_cast<long long *>(p), v); }
__device__ __forceinline__ void st_stream_4(void *p, int v) { __stcs(reinterpret_cast<int *>(p), v); }

__device__ __forceinline__ uint64_t l2_policy_evict_last() {
    uint64_t pol;
    asm volatile("createpolicy.fractional.L2::evict_last.b64 %0, 1.0;" : "=l"(pol));
    return pol;
}
__device__ __forceinline__ int4 ld_keep_16(const void *p, uint64_t pol) {
    int4 v;
    asm volatile("ld.global.nc.L2::cache_hint.v4.s32 {%0,%1,%2,%3}, [%4], %5;"
                 : "=r"(v.x), "=r"(v.y), "=r"(v.z), "=r"(v.w)
                 : "l"(p), "l"(pol));
    return v;
}
__device__ __forceinline__ int4 ld_keep_16_na(const void *p, uint64_t pol) {  // same, without allocating an L1 line
    int4 v;
    asm volatile("ld.global.nc.L1::no_allocate.L2::cache_hint.v4.s32 {%0,%1,%2,%3}, [%4], %5;"
                 : "=r"(v.x), "=r"(v.y), "=r"(v.z), "=r"(v.w)
                 : "l"(p), "l"(pol));
    return v;
}
__device__ __forceinline__ unsigned long long ld_keep_8(const void *p, uint64_t pol) {
    unsigned long long v;
    asm volatile("ld.global.nc.L2::cache_hint.u64 %0, [%1], %2;" : "=l"(v) : "l"(p), "l"(pol));
    return v;
}
__device__ __forceinline__ unsigned long long ld_keep_8_na(const void *p, uint64_t pol) {
    unsigned long long v;
    asm volatile("ld.global.nc.L1::no_allocate.L2::cache_hint.u64 %0, [%1], %2;" : "=l"(v) : "l"(p), "l"(pol));
    return v;
}
__device__ __forceinline__ unsigned int ld_keep_4(const void *p, uint64_t pol) {
    unsigned int v;
    asm volatile("ld.global.nc.L2::cache_hint.u32 %0, [%1], %2;" : "=r"(v) : "l"(p), "l"(pol));
    return v;
}

// fp64 / u64 reductions that keep their line in L2 with evict_last priority (group-by accumulators: a partition's slice of
// them is re-touched for millions of rows while the input streams by with evict-first loads)
__device__ __forceinline__ void red_add_f64_keep(double *p, double v, uint64_t pol) {
    asm volatile("red.global.add.L2::cache_hint.f64 [%0], %1, %2;" ::"l"(p), "d"(v), "l"(pol) : "memory");
}
__device__ __forceinline__ void red_add_u64_keep(unsigned long long *p, unsigned long long v, uint64_t pol) {
    asm volatile("red.global.add.L2::cache_hint.u64 [%0], %1, %2;" ::"l"(p), "l"(v), "l"(pol) : "memory");
}
__device__ __forceinline__ unsigned int ld_keep_u8(const uint8_t *p, uint64_t pol) {
    unsigned int v;
    asm volatile("ld.global.L2::cache_hint.u8 %0, [%1], %2;" : "=r"(v) : "l"(p), "l"(pol));
    return v;
}

// ---- cp.async (LDGSTS): per-thread asynchronous global -> shared copies, grouped and waited per tile.  The source must
// be naturally aligned.
__device__ __forceinline__ void cp_async_4(void *smem_dst, const void *gsrc) {
    asm volatile("cp.async.ca.shared.global [%0], [%1], 4;" ::"r"((uint32_t)__cvta_generic_to_shared(smem_dst)), "l"(gsrc) : "memory");
}
__device__ __forceinline__ void cp_async_8(void *smem_dst, const void *gsrc) {
    asm volatile("cp.async.ca.shared.global [%0], [%1], 8;" ::"r"((uint32_t)__cvta_generic_to_shared(smem_dst)), "l"(gsrc) : "memory");
}
__device__ __forceinline__ void cp_async_commit() { asm volatile("cp.async.commit_group;" ::: "memory"); }
template <int N>
__device__ __forceinline__ void cp_async_wait() { asm volatile("cp.async.wait_group %0;" ::"n"(N) : "memory"); }

// ---- mbarrier + 1-D bulk copy (cp.async.bulk; SASS: UBLKCP / SYNCS).  The uint32_t forms take shared-memory addresses,
// for kernels that compute them once instead of per call.
__device__ __forceinline__ uint32_t smem_u32(const void *p) { return (uint32_t)__cvta_generic_to_shared(p); }
__device__ __forceinline__ void mbar_init(unsigned long long *bar, int count) {
    asm volatile("mbarrier.init.shared::cta.b64 [%0], %1;" ::"r"(smem_u32(bar)), "r"(count) : "memory");
}
__device__ __forceinline__ void mbar_expect_tx(uint32_t bar, uint32_t bytes) {
    asm volatile("mbarrier.arrive.expect_tx.shared::cta.b64 _, [%0], %1;" ::"r"(bar), "r"(bytes) : "memory");
}
__device__ __forceinline__ void mbar_expect_tx(unsigned long long *bar, uint32_t bytes) { mbar_expect_tx(smem_u32(bar), bytes); }
__device__ __forceinline__ void mbar_arrive(uint32_t bar) { asm volatile("mbarrier.arrive.shared::cta.b64 _, [%0];" ::"r"(bar) : "memory"); }
__device__ __forceinline__ void mbar_wait(uint32_t bar, uint32_t parity) {
    uint32_t done = 0;
    while (!done)
        asm volatile("{\n\t.reg .pred p;\n\tmbarrier.try_wait.parity.shared::cta.b64 p, [%1], %2;\n\tselp.u32 %0, 1, 0, p;\n\t}"
                     : "=r"(done) : "r"(bar), "r"(parity) : "memory");
}
__device__ __forceinline__ void mbar_wait(unsigned long long *bar, uint32_t parity) { mbar_wait(smem_u32(bar), parity); }
__device__ __forceinline__ uint64_t l2_policy_evict_first() {
    uint64_t pol;
    asm volatile("createpolicy.fractional.L2::evict_first.b64 %0, 1.0;" : "=l"(pol));
    return pol;
}
// 1-D bulk copy global -> shared, completion signalled on an mbarrier; source, destination and size are multiples of 16 B
__device__ __forceinline__ void tma_load_1d(uint32_t smem_dst, const void *gsrc, uint32_t bytes, uint32_t bar, uint64_t pol) {
    asm volatile("cp.async.bulk.shared::cluster.global.mbarrier::complete_tx::bytes.L2::cache_hint [%0], [%1], %2, [%3], %4;" ::"r"(smem_dst),
                 "l"(gsrc), "r"(bytes), "r"(bar), "l"(pol)
                 : "memory");
}
__device__ __forceinline__ void tma_load_1d(void *smem_dst, const void *gsrc, uint32_t bytes, unsigned long long *bar, uint64_t pol) {
    tma_load_1d(smem_u32(smem_dst), gsrc, bytes, smem_u32(bar), pol);
}

static inline int64_t div_up(int64_t a, int64_t b) { return (a + b - 1) / b; }

// xchg.cu: reorders `rows` rows of up to 4 NULL-free device columns by destination = mulhi(fmix64(key), nparts) — the
// table-slot range of the group-by / join tables — with the warp-synchronous split kernels of the push exchange
// (nparts <= GSQL_MAX_RANKS).  out_data[c] receives column c; destinations are contiguous, in order.  Runs on ctx->stream.
gsql_status local_split_by_slot_range(gsql_ctx *ctx, const DColSet &in, int key_col, int64_t rows, int nparts, void *const *out_data);
