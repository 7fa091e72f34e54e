// bloom.cu — the join's runtime bloom filter behind gsql_bloom_* (xxhash_64 method only).
//
// Reference path replaced (COM/ = polardbx-common/src/main/java/com/alibaba/polardbx/common/,
// EX/ = polardbx-executor/src/main/java/com/alibaba/polardbx/executor/):
//   EX/operator/RuntimeFilterBuilderExec.java + EX/mpp/operator/BloomFilterProduce.addChunk:92-106 (build side: every key
//     row hashed into the filter), COM/utils/bloomfilter/BloomFilter.java:65-76 (put64), :114-129 (mightContain64),
//     :164-170 (merge), COM/utils/bloomfilter/BitSet.java:53-82 (bit i = data[i >>> 6] & (1L << (i & 63)))
//   EX/operator/FilterExec.java:81-130 with condition BLOOMFILTER(key) (probe side: rows that cannot match are dropped)
// The filter is observable across the exchange boundary — a filter built here is merged at the coordinator with filters
// from stock Java tasks and tested by the storage node — so the bits set are the reference's, bit for bit:
//   * the key is fed to the streaming hasher as one long (Chunk.ChunkRow.hashCode -> addToHasher): INT sign-extends
//     (IStreamingHasher.putInt -> putLong), BIGINT as is, DOUBLE as Double.doubleToRawLongBits (no NaN canonicalisation,
//     -0.0 != +0.0), NULL as the block's NULL_VALUE 0; for one long the streaming XXH64 is XXH64(seed 0) of its 8
//     little-endian bytes;
//   * h1 = (int) h, h2 = (int) (h >>> 32), combined = h1 + h2 (Java int wraparound: done in uint32_t here), then k times:
//     clear the sign bit if set, set / test bit combined % numBits, combined += h2.
// The modulo runs k times per row: it is Lemire's exact precomputed-reciprocal fastmod (one 64-bit multiply and one
// __umul64hi), exact for every 32-bit dividend and divisor, not a hardware divide.
#include "common.cuh"

namespace {

constexpr int BF_THREADS = 256;
constexpr int BF_RPT = 4;
constexpr int BF_TILE = BF_THREADS * BF_RPT;
constexpr int64_t BF_MAX_BITS = (int64_t)2147483647 - 63;  // BloomFilter.java:45 Math.multiplyExact(length, 64): 2^31 - 64

constexpr uint64_t XXP1 = 0x9E3779B185EBCA87ULL;
constexpr uint64_t XXP2 = 0xC2B2AE3D27D4EB4FULL;
constexpr uint64_t XXP3 = 0x165667B19E3779F9ULL;
constexpr uint64_t XXP4 = 0x85EBCA77C2B2AE63ULL;
constexpr uint64_t XXP5 = 0x27D4EB2F165667C5ULL;

__host__ __device__ __forceinline__ uint64_t rotl64(uint64_t x, int r) { return (x << r) | (x >> (64 - r)); }

// XXH64(seed = 0) of the 8 little-endian bytes of v: one 8-byte lane round, then the avalanche.
__host__ __device__ __forceinline__ uint64_t xxh64_u64(uint64_t v) {
    uint64_t h = XXP5 + 8;
    h ^= rotl64(v * XXP2, 31) * XXP1;
    h = rotl64(h, 27) * XXP1 + XXP4;
    h ^= h >> 33;
    h *= XXP2;
    h ^= h >> 29;
    h *= XXP3;
    h ^= h >> 32;
    return h;
}

// Lemire, Kaser, Kurz, "Faster remainder by direct computation" (2019): a % d for 32-bit a, d with M = 2^64 / d + 1.
__device__ __forceinline__ uint32_t fastmod_u32(uint32_t a, uint64_t M, uint32_t d) {
    return (uint32_t)__umul64hi(M * (uint64_t)a, (uint64_t)d);
}
static inline uint64_t fastmod_magic(uint32_t d) { return UINT64_C(0xFFFFFFFFFFFFFFFF) / d + 1; }

// The long the reference's hasher sees for row r of a key column.
__device__ __forceinline__ uint64_t key_long(const DCol &c, int64_t r) {
    if (c.nulls != nullptr && c.nulls[r] != 0) return 0;  // NULL_VALUE
    if (c.type == GSQL_T_INT32) return (uint64_t)(int64_t)ld_stream_4(reinterpret_cast<const int *>(c.data) + r);
    return (uint64_t)ld_stream_8(reinterpret_cast<const long long *>(c.data) + r);  // BIGINT, or DOUBLE raw bits
}

struct BloomGeom {
    uint64_t *words;
    uint64_t M;
    uint32_t nbits;
    int32_t k;
};

__global__ void __launch_bounds__(BF_THREADS) k_bloom_put(const __grid_constant__ DCol key, int64_t rows, const __grid_constant__ BloomGeom G) {
    for (int64_t r = blockIdx.x * (int64_t)blockDim.x + threadIdx.x; r < rows; r += (int64_t)gridDim.x * blockDim.x) {
        const uint64_t h = xxh64_u64(key_long(key, r));
        const uint32_t h2 = (uint32_t)(h >> 32);
        uint32_t c = (uint32_t)h + h2;
#pragma unroll 1
        for (int i = 0; i < G.k; i++) {
            c &= 0x7fffffffu;  // `if (combined < 0) combined &= MAX_VALUE` — a no-op on non-negative values
            const uint32_t bit = fastmod_u32(c, G.M, G.nbits);
            atomicOr(reinterpret_cast<unsigned long long *>(G.words) + (bit >> 6), 1ULL << (bit & 63));
            c += h2;
        }
    }
}

struct BloomOut {
    void *data[GSQL_MAX_COLS];
    uint8_t *nulls[GSQL_MAX_COLS];
};

// Probe side: tests the key of every row (stopping at the first clear bit, as mightContain64 does) and compacts the
// surviving rows of every column into `O`: warp ballots rank a 1024-row tile's survivors, one cursor bump reserves
// their output range (k_scan's scheme, scan.cu), so a tile's rows keep their input order and tiles land in cursor order.
__global__ void __launch_bounds__(BF_THREADS) k_bloom_filter(const __grid_constant__ DColSet in, int32_t key_col, int64_t rows,
                                                             const __grid_constant__ BloomGeom G, const __grid_constant__ BloomOut O,
                                                             unsigned long long *cursor, int32_t *flags) {
    __shared__ unsigned int wcount[BF_THREADS / 32][BF_RPT];
    __shared__ unsigned long long tile_base;
    const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
    const uint64_t pol = l2_policy_evict_last();  // the bitmap is re-read by every row: keep it in L2
    const int64_t ntiles = (rows + BF_TILE - 1) / BF_TILE;
    const DCol key = in.c[key_col];
    for (int64_t tile = blockIdx.x; tile < ntiles; tile += gridDim.x) {
        const int64_t t0 = tile * BF_TILE + threadIdx.x;  // this thread's row in slot 0; slot s is s * BF_THREADS further
        bool pass[BF_RPT];
        unsigned int ballot[BF_RPT];
#pragma unroll
        for (int s = 0; s < BF_RPT; s++) {
            const int64_t r = t0 + s * BF_THREADS;
            pass[s] = r < rows;
            if (!pass[s]) continue;
            const uint64_t h = xxh64_u64(key_long(key, r));
            const uint32_t h2 = (uint32_t)(h >> 32);
            uint32_t c = (uint32_t)h + h2;
#pragma unroll 1
            for (int i = 0; i < G.k; i++) {
                c &= 0x7fffffffu;
                const uint32_t bit = fastmod_u32(c, G.M, G.nbits);
                if (!((ld_keep_8(G.words + (bit >> 6), pol) >> (bit & 63)) & 1ULL)) {
                    pass[s] = false;
                    break;
                }
                c += h2;
            }
        }
#pragma unroll
        for (int s = 0; s < BF_RPT; s++) {
            ballot[s] = __ballot_sync(0xffffffffu, pass[s]);
            if (lane == 0) wcount[warp][s] = __popc(ballot[s]);
        }
        __syncthreads();
        if (warp == 0) {  // 32 cells: exclusive scan in (slot, warp) order keeps the tile's rows in input order
            const int s = lane / (BF_THREADS / 32), w = lane % (BF_THREADS / 32);
            const unsigned int cnt = wcount[w][s];
            unsigned int incl = cnt;
#pragma unroll
            for (int d = 1; d < 32; d <<= 1) {
                const unsigned int t = __shfl_up_sync(0xffffffffu, incl, d);
                if (lane >= d) incl += t;
            }
            const unsigned int total = __shfl_sync(0xffffffffu, incl, 31);
            wcount[w][s] = incl - cnt;
            if (lane == 0) tile_base = total ? atomicAdd(cursor, (unsigned long long)total) : 0ULL;
            static_assert((BF_THREADS / 32) * BF_RPT == 32, "cell scan assumes 32 cells");
        }
        __syncthreads();
        unsigned long long pos[BF_RPT];
#pragma unroll
        for (int s = 0; s < BF_RPT; s++) pos[s] = tile_base + wcount[warp][s] + __popc(ballot[s] & ((1u << lane) - 1u));
#pragma unroll 1
        for (int e = 0; e < in.n; e++) {
            const DCol c = in.c[e];
            const bool w4 = c.type == GSQL_T_INT32;
#pragma unroll
            for (int s = 0; s < BF_RPT; s++) {
                if (!pass[s]) continue;
                const int64_t r = t0 + s * BF_THREADS;
                if (w4) reinterpret_cast<int *>(O.data[e])[pos[s]] = ld_stream_4(reinterpret_cast<const int *>(c.data) + r);
                else reinterpret_cast<long long *>(O.data[e])[pos[s]] = ld_stream_8(reinterpret_cast<const long long *>(c.data) + r);
                const uint8_t n = c.nulls ? (c.nulls[r] != 0) : 0;
                if (O.nulls[e]) O.nulls[e][pos[s]] = n;
                else if (n) flags[0] = 1;
            }
        }
        __syncthreads();  // wcount / tile_base are rewritten by the next tile
    }
}

// dst[w] |= src[f * nwords + w] for every filter f: BloomFilter.merge (BitSet.putAll) of m filters at once.
__global__ void __launch_bounds__(BF_THREADS) k_bloom_or(const unsigned long long *__restrict__ src, int64_t nfilters, int64_t nwords,
                                                         unsigned long long *__restrict__ dst) {
    for (int64_t w = blockIdx.x * (int64_t)blockDim.x + threadIdx.x; w < nwords; w += (int64_t)gridDim.x * blockDim.x) {
        unsigned long long v = dst[w];
        for (int64_t f = 0; f < nfilters; f++) v |= __ldcs(src + f * nwords + w);
        dst[w] = v;
    }
}

}  // namespace

struct gsql_bloom {
    gsql_ctx *ctx;
    int64_t num_bits;
    int32_t k;
    uint64_t M;
    DevBuf words, cursor, flags;
    BloomGeom geom() const { return BloomGeom{words.as<uint64_t>(), M, (uint32_t)num_bits, k}; }
    int64_t nwords() const { return num_bits / 64; }
};

extern "C" gsql_status gsql_bloom_create(gsql_ctx *ctx, int64_t num_bits, int32_t num_hash_functions, gsql_bloom **out) {
    if (!ctx || !out) return GSQL_E_INVALID;
    *out = nullptr;
    if (ctx->sticky) return GSQL_E_CUDA;
    if (num_bits < 64 || num_bits % 64 != 0 || num_bits > BF_MAX_BITS)
        return gsql_set_error(ctx, GSQL_E_INVALID, "num_bits %lld: must be a multiple of 64 in [64, 2^31-64]", (long long)num_bits);
    if (num_hash_functions < 1) return gsql_set_error(ctx, GSQL_E_INVALID, "num_hash_functions %d < 1", num_hash_functions);
    if (num_hash_functions > 64) return gsql_set_error(ctx, GSQL_E_UNSUPPORTED, "num_hash_functions %d > 64", num_hash_functions);
    GSQL_CUDA(ctx, cudaSetDevice(ctx->device));
    gsql_bloom *b = new gsql_bloom();
    b->ctx = ctx;
    b->num_bits = num_bits;
    b->k = num_hash_functions;
    b->M = fastmod_magic((uint32_t)num_bits);
    gsql_status st = b->words.alloc(ctx, (size_t)num_bits / 8);
    if (st == GSQL_OK) st = b->cursor.alloc(ctx, 16);
    if (st == GSQL_OK) st = b->flags.alloc(ctx, 16);
    if (st == GSQL_OK && cudaMemsetAsync(b->words.p, 0, (size_t)num_bits / 8, ctx->stream) != cudaSuccess) st = GSQL_E_CUDA;
    if (st == GSQL_OK && cudaMemsetAsync(b->flags.p, 0, 16, ctx->stream) != cudaSuccess) st = GSQL_E_CUDA;
    if (st != GSQL_OK) { delete b; return st; }
    gsql_ctx_retain(ctx);
    *out = b;
    return GSQL_OK;
}

extern "C" void gsql_bloom_destroy(gsql_bloom *b) { destroy_handle(b); }

static gsql_status check_key(gsql_ctx *ctx, const gsql_batch *batch, int32_t key_col) {
    GSQL_TRY(validate_batch(ctx, batch, -1, nullptr));
    if (key_col < 0 || key_col >= batch->ncols) return gsql_set_error(ctx, GSQL_E_INVALID, "key column %d out of range", key_col);
    const int t = batch->cols[key_col].type;
    if (t != GSQL_T_INT32 && t != GSQL_T_INT64 && t != GSQL_T_FP64)
        return gsql_set_error(ctx, GSQL_E_UNSUPPORTED, "key column type %d: INT32, INT64 or FP64 only", t);
    return GSQL_OK;
}

extern "C" gsql_status gsql_bloom_put(gsql_bloom *b, const gsql_batch *batch, int32_t key_col) {
    if (!b || !batch) return GSQL_E_INVALID;
    gsql_ctx *ctx = b->ctx;
    if (ctx->sticky) return GSQL_E_CUDA;
    GSQL_TRY(check_key(ctx, batch, key_col));
    if (batch->rows == 0) return GSQL_OK;
    GSQL_CUDA(ctx, cudaSetDevice(ctx->device));
    gsql_col kc = batch->cols[key_col];  // only the key column is staged
    gsql_batch one = {batch->rows, 1, batch->mem, &kc};
    StagedBatch sb;
    GSQL_TRY(stage_batch(ctx, &one, &sb));
    {
        KernelScope ks(ctx, "k_bloom_put");
        k_bloom_put<<<grid_for(ctx, batch->rows, BF_THREADS, 8), BF_THREADS, 0, ctx->stream>>>(sb.cols[0], batch->rows, b->geom());
    }
    GSQL_CUDA(ctx, cudaGetLastError());
    if (batch->mem == GSQL_MEM_HOST) GSQL_CUDA(ctx, cudaStreamSynchronize(ctx->stream));  // staged copies die with `sb`
    return GSQL_OK;
}

extern "C" gsql_status gsql_bloom_merge(gsql_bloom *b, const uint64_t *words, int64_t nfilters, int32_t mem) {
    if (!b) return GSQL_E_INVALID;
    gsql_ctx *ctx = b->ctx;
    if (ctx->sticky) return GSQL_E_CUDA;
    if (nfilters < 0 || (nfilters > 0 && !words) || (mem != GSQL_MEM_HOST && mem != GSQL_MEM_DEVICE))
        return gsql_set_error(ctx, GSQL_E_INVALID, "bad merge arguments (nfilters %lld, mem %d)", (long long)nfilters, mem);
    if (nfilters == 0) return GSQL_OK;
    GSQL_CUDA(ctx, cudaSetDevice(ctx->device));
    const int64_t nw = b->nwords();
    DevBuf staged;
    const uint64_t *src = words;
    if (mem == GSQL_MEM_HOST) {
        GSQL_TRY(staged.alloc(ctx, (size_t)(nfilters * nw) * 8));
        GSQL_CUDA(ctx, cudaMemcpyAsync(staged.p, words, (size_t)(nfilters * nw) * 8, cudaMemcpyHostToDevice, ctx->stream));
        src = staged.as<uint64_t>();
    }
    {
        KernelScope ks(ctx, "k_bloom_or");
        k_bloom_or<<<grid_for(ctx, nw, BF_THREADS, 8), BF_THREADS, 0, ctx->stream>>>(reinterpret_cast<const unsigned long long *>(src), nfilters, nw,
                                                                              b->words.as<unsigned long long>());
    }
    GSQL_CUDA(ctx, cudaGetLastError());
    if (mem == GSQL_MEM_HOST) GSQL_CUDA(ctx, cudaStreamSynchronize(ctx->stream));
    return GSQL_OK;
}

extern "C" gsql_status gsql_bloom_bitmap(gsql_bloom *b, uint64_t *words, int32_t mem) {
    if (!b) return GSQL_E_INVALID;
    gsql_ctx *ctx = b->ctx;
    if (ctx->sticky) return GSQL_E_CUDA;
    if (!words || (mem != GSQL_MEM_HOST && mem != GSQL_MEM_DEVICE)) return gsql_set_error(ctx, GSQL_E_INVALID, "bad bitmap arguments");
    GSQL_CUDA(ctx, cudaSetDevice(ctx->device));
    GSQL_CUDA(ctx, cudaMemcpyAsync(words, b->words.p, (size_t)b->num_bits / 8,
                                   mem == GSQL_MEM_HOST ? cudaMemcpyDeviceToHost : cudaMemcpyDeviceToDevice, ctx->stream));
    if (mem == GSQL_MEM_HOST) GSQL_CUDA(ctx, cudaStreamSynchronize(ctx->stream));
    return GSQL_OK;
}

extern "C" gsql_status gsql_bloom_filter(gsql_bloom *b, const gsql_batch *in, int32_t key_col, gsql_batch *out, int64_t out_capacity,
                                         int64_t *out_rows) {
    if (!b || !in || !out || !out_rows) return GSQL_E_INVALID;
    gsql_ctx *ctx = b->ctx;
    if (ctx->sticky) return GSQL_E_CUDA;
    GSQL_TRY(check_key(ctx, in, key_col));
    int32_t types[GSQL_MAX_COLS];
    for (int i = 0; i < in->ncols; i++) types[i] = in->cols[i].type;
    GSQL_TRY(validate_batch(ctx, out, in->ncols, types));
    if (in->mem != out->mem) return gsql_set_error(ctx, GSQL_E_INVALID, "in and out must live in the same memory space");
    for (int i = 0; i < in->ncols; i++)
        if (types[i] == GSQL_T_DEC128) return gsql_set_error(ctx, GSQL_E_UNSUPPORTED, "column %d: DEC128 is output-only", i);
    *out_rows = 0;
    out->rows = 0;
    if (in->rows == 0) return GSQL_OK;
    if (out_capacity < in->rows) {
        *out_rows = in->rows;
        return gsql_set_error(ctx, GSQL_E_CAPACITY, "filter output must hold the input's %lld rows", (long long)in->rows);
    }
    GSQL_CUDA(ctx, cudaSetDevice(ctx->device));
    StagedBatch sb;
    GSQL_TRY(stage_batch(ctx, in, &sb));
    const DColSet cols = sb.set();
    OutBinding ob;
    GSQL_TRY(out_bind(ctx, out, in->rows, &ob));
    BloomOut O;
    memset(&O, 0, sizeof(O));
    for (int e = 0; e < in->ncols; e++) {
        O.data[e] = ob.data[e];
        O.nulls[e] = ob.nulls[e];
    }
    GSQL_CUDA(ctx, cudaMemsetAsync(b->cursor.p, 0, 16, ctx->stream));
    {
        KernelScope ks(ctx, "k_bloom_filter");
        k_bloom_filter<<<grid_for(ctx, in->rows, BF_TILE, 8), BF_THREADS, 0, ctx->stream>>>(cols, key_col, in->rows, b->geom(), O,
                                                                                      b->cursor.as<unsigned long long>(), b->flags.as<int32_t>());
    }
    GSQL_CUDA(ctx, cudaGetLastError());
    struct { unsigned long long n; unsigned long long pad; } h;
    int32_t hf[4];
    GSQL_CUDA(ctx, cudaMemcpyAsync(&h, b->cursor.p, 16, cudaMemcpyDeviceToHost, ctx->stream));
    GSQL_CUDA(ctx, cudaMemcpyAsync(hf, b->flags.p, 16, cudaMemcpyDeviceToHost, ctx->stream));
    GSQL_CUDA(ctx, cudaStreamSynchronize(ctx->stream));
    if (hf[0]) {
        cudaMemsetAsync(b->flags.p, 0, 16, ctx->stream);
        return gsql_set_error(ctx, GSQL_E_INVALID, "a NULL had to be written into an output column without a nulls buffer");
    }
    const int64_t n = (int64_t)h.n;
    GSQL_TRY(out_download(ctx, out, n, ob));
    *out_rows = out->rows = n;
    return GSQL_OK;
}
