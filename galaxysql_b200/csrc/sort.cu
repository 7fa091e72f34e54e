// sort.cu — ORDER BY and ORDER BY ... LIMIT behind gsql_sort_* (SortExec / MemSortor and SpilledTopNExec), and the merge
// of pre-sorted runs behind gsql_merge_* (MergeSortExec; its own section at the end of the file).
//
// Reference path replaced (EX/ = polardbx-executor/src/main/java/com/alibaba/polardbx/executor/,
// OPT/ = polardbx-optimizer/src/main/java/com/alibaba/polardbx/optimizer/):
//   EX/operator/SortExec.java + EX/operator/util/MemSortor.java:60-78 (IntArrays.quickSort of row positions)
//   EX/operator/SpilledTopNExec.java:66-70 (topSize = skip + fetch; 0 outputs nothing, < 0 is an error)
// Row order is the executor's comparator, EX/utils/ExecUtils.getComparator:451-490, bit for bit:
//   * keys compare in order; two NULLs are equal and NULL is the smallest value (OPT/core/datatype/NumberType.compare:110-127);
//     DESC negates the result, so NULLs come first under ASC and last under DESC (the collation's nullLast is never read);
//   * INT / BIGINT (and DATE, which reaches the executor as a packed BIGINT) in natural order; DOUBLE by Double.compareTo:
//     -0.0 < +0.0, every NaN payload is one value, above +Inf;
//   * ties are unordered (quickSort is not stable), and so is the choice among rows tied at a TopN boundary.
//
// Every key becomes an unsigned field whose integer order is that order: the value's order-preserving u64 image minus the
// minimum image over the rows being ordered (k_sort_minmax), in ceil(log2(range + 1)) bits, under a NULL bit when a NULL
// is present, complemented under DESC.  Fields are packed most significant key first into groups of at most 128 bits.
// A full sort radix-sorts (row id, group image) pairs with cub, least significant group first: cub's sort is stable, so
// each later group refines the permutation the earlier ones left.  A TopN radix-selects on the leading group (11-bit digit
// histogram, threshold picked on the device, ballot compaction of the row ids at or below it) until at most ~4 L candidates
// remain, then sorts just those.  Consumed batches are cut to their best L rows as they arrive, so a TopN holds O(L) rows.
#include <cub/device/device_radix_sort.cuh>
#include <cub/block/block_scan.cuh>
#include <cuda/std/tuple>

#include "common.cuh"

namespace {

constexpr int SO_THREADS = 256;
constexpr int SO_RPT = 4;
constexpr int SO_TILE = SO_THREADS * SO_RPT;
constexpr int DIGIT_BITS = 11;
constexpr int NBINS = 1 << DIGIT_BITS;
constexpr int64_t MAX_ROW_IDS = INT32_MAX;  // row ids are 32-bit and cub's item count is an int
constexpr int64_t TOPN_SLICE = (int64_t)1 << 30;
constexpr int64_t TOPN_REFINE_FACTOR = 4;   // refine the selection while candidates exceed this many times the limit
constexpr int64_t TOPN_HOLD_MIN = 1 << 16;  // held rows may grow to max(2 L, this) before they are cut back to L
// A top-n holds at most max(2 L, TOPN_HOLD_MIN) + L rows (the bound, plus one batch's best L) and selects over them with
// 32-bit row ids; a larger limit holds every row like a full sort, under the full sort's capacity check.
constexpr int64_t TOPN_MAX_LIMIT = (MAX_ROW_IDS - TOPN_HOLD_MIN) / 3;

typedef unsigned __int128 u128;

struct K128 {  // a group image as cub sees it: two 64-bit digits, `hi` most significant
    uint64_t lo, hi;
};
struct K128Decomposer {
    __host__ __device__ cuda::std::tuple<uint64_t &, uint64_t &> operator()(K128 &k) const { return {k.hi, k.lo}; }
};

__device__ __forceinline__ u128 shr128(u128 x, int s) { return s >= 128 ? (u128)0 : (x >> s); }

struct KeyCols {
    int32_t n;
    int32_t pad;
    DCol c[GSQL_MAX_KEYS];
};

struct MinMax {  // over the non-NULL rows of each key; has_null[k] != 0 when key k holds a NULL
    unsigned long long mn[GSQL_MAX_KEYS], mx[GSQL_MAX_KEYS];
    unsigned int has_null[GSQL_MAX_KEYS];
};

// Order-preserving unsigned image of a non-NULL value: sign flip for integers; for doubles NaN is canonicalised and
// negative values are complemented, positive ones get the sign bit, so -0.0 < +0.0 and NaN sits above +Inf.
__device__ __forceinline__ uint64_t value_image(const DCol &c, int64_t r) {
    if (c.type == GSQL_T_INT32) return (uint64_t)(int64_t)ld_stream_4(reinterpret_cast<const int *>(c.data) + r) ^ (1ULL << 63);
    const uint64_t b = (uint64_t)ld_stream_8(reinterpret_cast<const long long *>(c.data) + r);
    if (c.type == GSQL_T_INT64) return b ^ (1ULL << 63);
    const uint64_t canon = ((b & 0x7fffffffffffffffULL) > 0x7ff0000000000000ULL) ? 0x7ff8000000000000ULL : b;
    return (canon >> 63) ? ~canon : (canon | (1ULL << 63));
}

__device__ __forceinline__ bool is_null(const DCol &c, int64_t r) { return c.nulls != nullptr && c.nulls[r] != 0; }

// One pass over the rows (all of them, or the `idx` list): per key the min / max image of the non-NULL rows and whether a
// NULL occurs.  Warp and block reductions, then one atomic per block per key and quantity.
__global__ void __launch_bounds__(SO_THREADS) k_sort_minmax(const __grid_constant__ KeyCols K, const uint32_t *__restrict__ idx,
                                                            int64_t n, MinMax *__restrict__ out) {
    __shared__ unsigned long long smn[SO_THREADS / 32], smx[SO_THREADS / 32];
    __shared__ unsigned int snl[SO_THREADS / 32];
    const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
#pragma unroll 1
    for (int k = 0; k < K.n; k++) {
        const DCol c = K.c[k];
        unsigned long long mn = ~0ULL, mx = 0;
        unsigned int nl = 0;
        for (int64_t i = blockIdx.x * (int64_t)blockDim.x + threadIdx.x; i < n; i += (int64_t)gridDim.x * blockDim.x) {
            const int64_t r = idx ? (int64_t)idx[i] : i;
            if (is_null(c, r)) {
                nl = 1;
                continue;
            }
            const unsigned long long v = value_image(c, r);
            mn = v < mn ? v : mn;
            mx = v > mx ? v : mx;
        }
#pragma unroll
        for (int d = 16; d > 0; d >>= 1) {
            const unsigned long long a = __shfl_xor_sync(0xffffffffu, mn, d), b = __shfl_xor_sync(0xffffffffu, mx, d);
            mn = a < mn ? a : mn;
            mx = b > mx ? b : mx;
        }
        nl = __any_sync(0xffffffffu, nl) ? 1u : 0u;
        if (lane == 0) smn[warp] = mn, smx[warp] = mx, snl[warp] = nl;
        __syncthreads();
        if (threadIdx.x == 0) {
            for (int w = 1; w < SO_THREADS / 32; w++) {
                mn = smn[w] < mn ? smn[w] : mn;
                mx = smx[w] > mx ? smx[w] : mx;
                nl |= snl[w];
            }
            if (mn <= mx) {
                atomicMin(&out->mn[k], mn);
                atomicMax(&out->mx[k], mx);
            }
            if (nl) atomicOr(&out->has_null[k], 1u);
        }
        __syncthreads();
    }
}

struct KeyEnc {
    DCol col;
    unsigned long long min;
    int32_t vbits;    // value bits: ceil(log2(max - min + 1))
    int32_t nullbit;  // 1: a NULL bit sits above the value (the rows hold a NULL)
    int32_t desc;
    int32_t shift;    // position of the field's least significant bit inside the group image
};

struct GroupEnc {
    int32_t nk;
    int32_t bits;  // used bits of the group image
    KeyEnc k[GSQL_MAX_KEYS];
};

__device__ __forceinline__ u128 group_image(const GroupEnc &G, int64_t r) {
    u128 img = 0;
#pragma unroll 1
    for (int k = 0; k < G.nk; k++) {
        const KeyEnc &e = G.k[k];
        u128 f = 0;
        if (!is_null(e.col, r)) {
            f = (u128)(value_image(e.col, r) - e.min);
            if (e.nullbit) f |= (u128)1 << e.vbits;
        }
        if (e.desc) f = ~f & (((u128)1 << (e.vbits + e.nullbit)) - 1);
        img |= f << e.shift;
    }
    return img;
}

__device__ __forceinline__ void store_key(uint32_t *p, u128 v) { *p = (uint32_t)v; }
__device__ __forceinline__ void store_key(uint64_t *p, u128 v) { *p = (uint64_t)v; }
__device__ __forceinline__ void store_key(K128 *p, u128 v) { *p = K128{(uint64_t)v, (uint64_t)(v >> 64)}; }

// keys[i] = image of row perm[i] (row i without a permutation), vals[i] = that row.
template <typename K>
__global__ void __launch_bounds__(SO_THREADS) k_sort_encode(const __grid_constant__ GroupEnc G, const uint32_t *__restrict__ perm, int64_t n,
                                                            K *__restrict__ keys, uint32_t *__restrict__ vals) {
    for (int64_t i = blockIdx.x * (int64_t)blockDim.x + threadIdx.x; i < n; i += (int64_t)gridDim.x * blockDim.x) {
        const uint32_t r = perm ? perm[i] : (uint32_t)i;
        store_key(keys + i, group_image(G, r));
        vals[i] = r;
    }
}

__global__ void __launch_bounds__(SO_THREADS) k_sort_iota(uint32_t *__restrict__ out, int64_t n) {
    for (int64_t i = blockIdx.x * (int64_t)blockDim.x + threadIdx.x; i < n; i += (int64_t)gridDim.x * blockDim.x) out[i] = (uint32_t)i;
}

// The selection's running state: every candidate's image agrees with `prefix` above bit `shift + digit bits` or is below
// it; `definite` candidates are strictly below (they are in the result), `need` more must come from the ones that agree.
struct TopnState {
    unsigned long long p_lo, p_hi;
    unsigned long long need, definite;
};

// Digit histogram of the candidates whose image agrees with the prefix: counts in shared memory, one global add per
// non-empty bin per CTA.
__global__ void __launch_bounds__(SO_THREADS) k_topn_hist(const __grid_constant__ GroupEnc G, const uint32_t *__restrict__ idx, int64_t n,
                                                          int shift, int dbits, const TopnState *__restrict__ st,
                                                          unsigned int *__restrict__ hist) {
    __shared__ unsigned int sh[NBINS];
    for (int b = threadIdx.x; b < NBINS; b += blockDim.x) sh[b] = 0;
    __syncthreads();
    const u128 prefix = ((u128)st->p_hi << 64) | st->p_lo;
    const unsigned int dmask = (1u << dbits) - 1u;
    for (int64_t i = blockIdx.x * (int64_t)blockDim.x + threadIdx.x; i < n; i += (int64_t)gridDim.x * blockDim.x) {
        const int64_t r = idx ? (int64_t)idx[i] : i;
        const u128 img = group_image(G, r);
        if (shr128(img, shift + dbits) != prefix) continue;
        atomicAdd(&sh[(unsigned int)(img >> shift) & dmask], 1u);
    }
    __syncthreads();
    for (int b = threadIdx.x; b < NBINS; b += blockDim.x)
        if (sh[b]) atomicAdd(&hist[b], sh[b]);
}

// One CTA: the smallest digit t whose inclusive count reaches `need`; the prefix gains t, the rows below t become definite.
// Clears the histogram for the next level.
constexpr int PICK_PER_THREAD = NBINS / SO_THREADS;
__global__ void __launch_bounds__(SO_THREADS) k_topn_pick(unsigned int *__restrict__ hist, int dbits, TopnState *__restrict__ st) {
    typedef cub::BlockScan<unsigned long long, SO_THREADS> Scan;
    __shared__ typename Scan::TempStorage tmp;
    unsigned long long local[PICK_PER_THREAD], sum = 0;
#pragma unroll
    for (int j = 0; j < PICK_PER_THREAD; j++) {
        local[j] = hist[threadIdx.x * PICK_PER_THREAD + j];
        hist[threadIdx.x * PICK_PER_THREAD + j] = 0;
        sum += local[j];
    }
    unsigned long long base;
    Scan(tmp).ExclusiveSum(sum, base);
    const unsigned long long need = st->need;
    __syncthreads();  // every thread has read `need` before the winner rewrites it
    if (base < need && need <= base + sum) {
        unsigned long long c = base;
#pragma unroll
        for (int j = 0; j < PICK_PER_THREAD; j++) {
            if (c + local[j] >= need) {
                const u128 p = ((((u128)st->p_hi << 64) | st->p_lo) << dbits) | (u128)(threadIdx.x * PICK_PER_THREAD + j);
                st->p_lo = (unsigned long long)p;
                st->p_hi = (unsigned long long)(p >> 64);
                st->definite += c;
                st->need = need - c;
                break;
            }
            c += local[j];
        }
    }
}

// Ballot compaction of the candidates whose image is at or below the prefix: warp ballots rank a tile's survivors and one
// cursor bump per tile reserves their range (k_bloom_filter's scheme).
__global__ void __launch_bounds__(SO_THREADS) k_topn_compact(const __grid_constant__ GroupEnc G, const uint32_t *__restrict__ idx, int64_t n,
                                                             int shift, const TopnState *__restrict__ st, uint32_t *__restrict__ out,
                                                             unsigned long long *__restrict__ cursor) {
    __shared__ unsigned int wcount[SO_THREADS / 32][SO_RPT];
    __shared__ unsigned long long tile_base;
    const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
    const u128 prefix = ((u128)st->p_hi << 64) | st->p_lo;
    const int64_t ntiles = (n + SO_TILE - 1) / SO_TILE;
    for (int64_t tile = blockIdx.x; tile < ntiles; tile += gridDim.x) {
        const int64_t t0 = tile * SO_TILE + threadIdx.x;
        bool keep[SO_RPT];
        uint32_t row[SO_RPT];
        unsigned int ballot[SO_RPT];
#pragma unroll
        for (int s = 0; s < SO_RPT; s++) {
            const int64_t i = t0 + s * SO_THREADS;
            keep[s] = false;
            row[s] = 0;
            if (i < n) {
                row[s] = idx ? idx[i] : (uint32_t)i;
                keep[s] = shr128(group_image(G, row[s]), shift) <= prefix;
            }
            ballot[s] = __ballot_sync(0xffffffffu, keep[s]);
            if (lane == 0) wcount[warp][s] = __popc(ballot[s]);
        }
        __syncthreads();
        if (warp == 0) {
            const int s = lane / (SO_THREADS / 32), w = lane % (SO_THREADS / 32);
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
            static_assert((SO_THREADS / 32) * SO_RPT == 32, "cell scan assumes 32 cells");
        }
        __syncthreads();
#pragma unroll
        for (int s = 0; s < SO_RPT; s++)
            if (keep[s]) out[tile_base + wcount[warp][s] + __popc(ballot[s] & ((1u << lane) - 1u))] = row[s];
        __syncthreads();
    }
}

struct GatherOut {
    void *data[GSQL_MAX_COLS];
    uint8_t *nulls[GSQL_MAX_COLS];
};

// out row i = source row perm[base + i] (row base + i without a permutation), every column with its NULL byte.  A NULL
// bound for a column without a NULL buffer raises flags[0].
__global__ void __launch_bounds__(SO_THREADS) k_sort_gather(const __grid_constant__ DColSet src, const uint32_t *__restrict__ perm, int64_t base,
                                                            int64_t n, const __grid_constant__ GatherOut O, int32_t *__restrict__ flags) {
    for (int64_t i = blockIdx.x * (int64_t)blockDim.x + threadIdx.x; i < n; i += (int64_t)gridDim.x * blockDim.x) {
        const int64_t r = perm ? (int64_t)perm[base + i] : base + i;
#pragma unroll 1
        for (int e = 0; e < src.n; e++) {
            const DCol c = src.c[e];
            if (c.type == GSQL_T_INT32) reinterpret_cast<int *>(O.data[e])[i] = reinterpret_cast<const int *>(c.data)[r];
            else reinterpret_cast<long long *>(O.data[e])[i] = reinterpret_cast<const long long *>(c.data)[r];
            const uint8_t nb = c.nulls ? (c.nulls[r] != 0) : 0;
            if (O.nulls[e]) O.nulls[e][i] = nb;
            else if (nb) flags[0] = 1;
        }
    }
}

int grid_of(gsql_ctx *ctx, int64_t items, int per_block) {
    const int64_t blocks = div_up(items, per_block), cap = (int64_t)ctx->sm_count * 8;
    return (int)(blocks < 1 ? 1 : (blocks < cap ? blocks : cap));
}

// Rows the handle holds, column-wise in HBM.  A column gets a NULL buffer once a batch with a mask arrives.
struct Held {
    int64_t rows = 0, cap = 0;
    int32_t ncols = 0;
    int32_t types[GSQL_MAX_COLS];
    DevBuf data[GSQL_MAX_COLS], nulls[GSQL_MAX_COLS];
    bool has_nulls[GSQL_MAX_COLS] = {};

    DColSet view() const {
        DColSet s;
        memset(&s, 0, sizeof(s));
        s.n = ncols;
        for (int e = 0; e < ncols; e++) s.c[e] = DCol{data[e].p, has_nulls[e] ? nulls[e].as<uint8_t>() : nullptr, types[e], 0};
        return s;
    }
};

}  // namespace

struct gsql_sort {
    gsql_ctx *ctx;
    gsql_sort_spec spec;
    bool topn;  // limit >= 0 and small enough to be selected; otherwise every row is held and sorted
    Held held;
    DevBuf perm;  // output order after finish: perm[i] = held row of output row i
    int64_t out_rows = 0, cursor = 0;
    bool finished = false;
    DevBuf mm, hist, state, cur, flags, temp;
    KeyCols keys_of(const DColSet &src) const {
        KeyCols k;
        memset(&k, 0, sizeof(k));
        k.n = spec.nkeys;
        for (int i = 0; i < spec.nkeys; i++) k.c[i] = src.c[spec.key_col[i]];
        return k;
    }
};

namespace {

// Key encodings grouped into <= 128-bit images, most significant group first (zero-width keys are dropped: all equal).
gsql_status plan_groups(gsql_sort *s, const DColSet &src, const uint32_t *idx, int64_t n, std::vector<GroupEnc> *groups) {
    gsql_ctx *ctx = s->ctx;
    MinMax h;
    memset(&h, 0, sizeof(h));
    for (int k = 0; k < GSQL_MAX_KEYS; k++) h.mn[k] = ~0ULL;
    GSQL_CUDA(ctx, cudaMemcpyAsync(s->mm.p, &h, sizeof(h), cudaMemcpyHostToDevice, ctx->stream));
    const KeyCols K = s->keys_of(src);
    {
        KernelScope ks(ctx, "k_sort_minmax");
        k_sort_minmax<<<grid_of(ctx, n, SO_THREADS * 8), SO_THREADS, 0, ctx->stream>>>(K, idx, n, s->mm.as<MinMax>());
    }
    GSQL_CUDA(ctx, cudaGetLastError());
    GSQL_CUDA(ctx, cudaMemcpyAsync(&h, s->mm.p, sizeof(h), cudaMemcpyDeviceToHost, ctx->stream));
    GSQL_CUDA(ctx, cudaStreamSynchronize(ctx->stream));
    groups->clear();
    GroupEnc g;
    memset(&g, 0, sizeof(g));
    std::vector<int> widths;
    auto close_group = [&]() {
        if (g.nk == 0) return;
        int at = g.bits;  // most significant key first
        for (int i = 0; i < g.nk; i++) {
            at -= g.k[i].vbits + g.k[i].nullbit;
            g.k[i].shift = at;
        }
        groups->push_back(g);
        memset(&g, 0, sizeof(g));
    };
    for (int k = 0; k < s->spec.nkeys; k++) {
        KeyEnc e;
        memset(&e, 0, sizeof(e));
        e.col = K.c[k];
        e.desc = s->spec.key_desc[k] != 0;
        e.nullbit = h.has_null[k] && h.mn[k] <= h.mx[k] ? 1 : 0;  // all NULL: the key is constant, no bit
        if (h.mn[k] <= h.mx[k]) {
            e.min = h.mn[k];
            const unsigned long long range = h.mx[k] - h.mn[k];
            e.vbits = range == 0 ? 0 : 64 - __builtin_clzll(range);
        }
        const int w = e.vbits + e.nullbit;
        if (w == 0) continue;
        if (g.bits + w > 128) close_group();
        g.k[g.nk++] = e;
        g.bits += w;
    }
    close_group();
    return GSQL_OK;
}

template <typename K>
gsql_status radix_group(gsql_sort *s, const GroupEnc &g, const uint32_t *perm_in, int64_t n, void *kbuf0, void *kbuf1, uint32_t *vals_in,
                        uint32_t *vals_out) {
    gsql_ctx *ctx = s->ctx;
    K *k0 = reinterpret_cast<K *>(kbuf0), *k1 = reinterpret_cast<K *>(kbuf1);
    {
        KernelScope ks(ctx, "k_sort_encode");
        k_sort_encode<K><<<grid_of(ctx, n, SO_THREADS), SO_THREADS, 0, ctx->stream>>>(g, perm_in, n, k0, vals_in);
    }
    GSQL_CUDA(ctx, cudaGetLastError());
    size_t need = 0;
    const int items = (int)n;
    if constexpr (sizeof(K) == 16) {
        GSQL_CUDA(ctx, cub::DeviceRadixSort::SortPairs(nullptr, need, k0, k1, vals_in, vals_out, items, K128Decomposer{}, 0, g.bits, ctx->stream));
    } else {
        GSQL_CUDA(ctx, cub::DeviceRadixSort::SortPairs(nullptr, need, k0, k1, vals_in, vals_out, items, 0, g.bits, ctx->stream));
    }
    if (!s->temp.p || need > s->temp.bytes) GSQL_TRY(s->temp.alloc(ctx, need));  // a null temp pointer would make cub only size
    need = s->temp.bytes;
    {
        KernelScope ks(ctx, "k_sort_radix");
        if constexpr (sizeof(K) == 16) {
            GSQL_CUDA(ctx, cub::DeviceRadixSort::SortPairs(s->temp.p, need, k0, k1, vals_in, vals_out, items, K128Decomposer{}, 0, g.bits,
                                                           ctx->stream));
        } else {
            GSQL_CUDA(ctx, cub::DeviceRadixSort::SortPairs(s->temp.p, need, k0, k1, vals_in, vals_out, items, 0, g.bits, ctx->stream));
        }
    }
    return GSQL_OK;
}

// out (n row ids) = the rows `idx` (all n rows of src without a list) in the comparator's order.
gsql_status sort_rows(gsql_sort *s, const DColSet &src, const uint32_t *idx, int64_t n, DevBuf *out) {
    gsql_ctx *ctx = s->ctx;
    GSQL_TRY(out->alloc(ctx, (size_t)n * 4));
    if (n == 0) return GSQL_OK;
    if (n > MAX_ROW_IDS)  // callers keep within this; cub's item count is an int
        return gsql_set_error(ctx, GSQL_E_CAPACITY, "%lld rows to sort exceed the 32-bit row ids", (long long)n);
    std::vector<GroupEnc> groups;
    GSQL_TRY(plan_groups(s, src, idx, n, &groups));
    if (groups.empty()) {  // every key is constant over these rows: any order is sorted
        if (idx) {
            GSQL_CUDA(ctx, cudaMemcpyAsync(out->p, idx, (size_t)n * 4, cudaMemcpyDeviceToDevice, ctx->stream));
        } else {
            KernelScope ks(ctx, "k_sort_iota");
            k_sort_iota<<<grid_of(ctx, n, SO_THREADS), SO_THREADS, 0, ctx->stream>>>(out->as<uint32_t>(), n);
        }
        GSQL_CUDA(ctx, cudaGetLastError());
        return GSQL_OK;
    }
    int kbytes = 4;
    for (const GroupEnc &g : groups) kbytes = g.bits > 64 ? 16 : (g.bits > 32 && kbytes < 8 ? 8 : kbytes);
    DevBuf k0, k1, v0, v1;
    GSQL_TRY(k0.alloc(ctx, (size_t)n * kbytes));
    GSQL_TRY(k1.alloc(ctx, (size_t)n * kbytes));
    GSQL_TRY(v0.alloc(ctx, (size_t)n * 4));
    GSQL_TRY(v1.alloc(ctx, (size_t)n * 4));
    // Least significant group first; cub's sort is stable, so each group refines the order the previous ones left.  The
    // encode copies the current permutation into v0 (element i is read before it is written), the sort writes v1 (or `out`).
    const uint32_t *perm = idx;
    for (int gi = (int)groups.size() - 1; gi >= 0; gi--) {
        uint32_t *vout = gi == 0 ? out->as<uint32_t>() : v1.as<uint32_t>();
        const GroupEnc &g = groups[gi];
        if (g.bits > 64) GSQL_TRY(radix_group<K128>(s, g, perm, n, k0.p, k1.p, v0.as<uint32_t>(), vout));
        else if (g.bits > 32) GSQL_TRY(radix_group<uint64_t>(s, g, perm, n, k0.p, k1.p, v0.as<uint32_t>(), vout));
        else GSQL_TRY(radix_group<uint32_t>(s, g, perm, n, k0.p, k1.p, v0.as<uint32_t>(), vout));
        perm = vout;
    }
    return GSQL_OK;
}

// out (*out_n = min(limit, n) row ids) = the first `limit` rows of src's n rows in the comparator's order.
gsql_status topn_rows(gsql_sort *s, const DColSet &src, int64_t n, int64_t limit, DevBuf *out, int64_t *out_n) {
    gsql_ctx *ctx = s->ctx;
    if (n <= limit) {
        *out_n = n;
        return sort_rows(s, src, nullptr, n, out);
    }
    *out_n = limit;
    if (limit == 0) return out->alloc(ctx, 16);
    if (n > MAX_ROW_IDS) return gsql_set_error(ctx, GSQL_E_CAPACITY, "%lld rows to select from exceed the 32-bit row ids", (long long)n);
    std::vector<GroupEnc> groups;
    GSQL_TRY(plan_groups(s, src, nullptr, n, &groups));
    if (groups.empty()) {  // all rows tie: any `limit` of them
        GSQL_TRY(out->alloc(ctx, (size_t)limit * 4));
        KernelScope ks(ctx, "k_sort_iota");
        k_sort_iota<<<grid_of(ctx, limit, SO_THREADS), SO_THREADS, 0, ctx->stream>>>(out->as<uint32_t>(), limit);
        GSQL_CUDA(ctx, cudaGetLastError());
        return GSQL_OK;
    }
    const GroupEnc &g0 = groups[0];
    TopnState h0 = {0, 0, (unsigned long long)limit, 0};
    GSQL_CUDA(ctx, cudaMemcpyAsync(s->state.p, &h0, sizeof(h0), cudaMemcpyHostToDevice, ctx->stream));
    GSQL_CUDA(ctx, cudaMemsetAsync(s->hist.p, 0, NBINS * 4, ctx->stream));
    DevBuf lists[2];
    const uint32_t *idx = nullptr;
    int64_t m = n;
    int hi = g0.bits, which = 0;
    while (true) {
        const int dbits = hi < DIGIT_BITS ? hi : DIGIT_BITS, shift = hi - dbits;
        {
            KernelScope ks(ctx, "k_topn_hist");
            k_topn_hist<<<grid_of(ctx, m, SO_THREADS * 8), SO_THREADS, 0, ctx->stream>>>(g0, idx, m, shift, dbits, s->state.as<TopnState>(),
                                                                                      s->hist.as<unsigned int>());
        }
        GSQL_CUDA(ctx, cudaGetLastError());
        {
            KernelScope ks(ctx, "k_topn_pick");
            k_topn_pick<<<1, SO_THREADS, 0, ctx->stream>>>(s->hist.as<unsigned int>(), dbits, s->state.as<TopnState>());
        }
        GSQL_CUDA(ctx, cudaGetLastError());
        DevBuf &dst = lists[which];
        GSQL_TRY(dst.alloc(ctx, (size_t)m * 4));
        GSQL_CUDA(ctx, cudaMemsetAsync(s->cur.p, 0, 8, ctx->stream));
        {
            KernelScope ks(ctx, "k_topn_compact");
            k_topn_compact<<<grid_of(ctx, m, SO_TILE), SO_THREADS, 0, ctx->stream>>>(g0, idx, m, shift, s->state.as<TopnState>(),
                                                                                     dst.as<uint32_t>(), s->cur.as<unsigned long long>());
        }
        GSQL_CUDA(ctx, cudaGetLastError());
        unsigned long long got = 0;
        GSQL_CUDA(ctx, cudaMemcpyAsync(&got, s->cur.p, 8, cudaMemcpyDeviceToHost, ctx->stream));
        GSQL_CUDA(ctx, cudaStreamSynchronize(ctx->stream));
        if ((int64_t)got < limit || (int64_t)got > m)
            return gsql_set_error(ctx, GSQL_E_CUDA, "top-n selection kept %llu of %lld rows for limit %lld", got, (long long)m, (long long)limit);
        idx = dst.as<uint32_t>();
        m = (int64_t)got;
        hi = shift;
        which ^= 1;
        lists[which].release();  // the list this level read
        if (m <= TOPN_REFINE_FACTOR * limit || hi == 0) break;
    }
    DevBuf sorted;
    GSQL_TRY(sort_rows(s, src, idx, m, &sorted));
    GSQL_TRY(out->alloc(ctx, (size_t)limit * 4));
    GSQL_CUDA(ctx, cudaMemcpyAsync(out->p, sorted.p, (size_t)limit * 4, cudaMemcpyDeviceToDevice, ctx->stream));
    return GSQL_OK;
}

// Appends rows perm[0..n) of src (rows 0..n without a permutation) to `h`.
gsql_status held_append(gsql_sort *s, Held *h, const DColSet &src, const uint32_t *perm, int64_t n) {
    gsql_ctx *ctx = s->ctx;
    if (n == 0) return GSQL_OK;
    const int64_t need = h->rows + n;
    if (need > h->cap) {
        int64_t cap = h->cap ? h->cap : 1024;
        while (cap < need) cap *= 2;
        for (int e = 0; e < h->ncols; e++) {
            GSQL_TRY(h->data[e].grow(ctx, (size_t)cap * gsql_type_width(h->types[e]), (size_t)h->rows * gsql_type_width(h->types[e])));
            if (h->has_nulls[e]) GSQL_TRY(h->nulls[e].grow(ctx, (size_t)cap, (size_t)h->rows));
        }
        h->cap = cap;
    }
    GatherOut O;
    memset(&O, 0, sizeof(O));
    for (int e = 0; e < h->ncols; e++) {
        if (src.c[e].nulls && !h->has_nulls[e]) {
            GSQL_TRY(h->nulls[e].alloc(ctx, (size_t)h->cap));
            GSQL_CUDA(ctx, cudaMemsetAsync(h->nulls[e].p, 0, (size_t)h->rows, ctx->stream));
            h->has_nulls[e] = true;
        }
        O.data[e] = h->data[e].as<char>() + (size_t)h->rows * gsql_type_width(h->types[e]);
        O.nulls[e] = h->has_nulls[e] ? h->nulls[e].as<uint8_t>() + h->rows : nullptr;
    }
    {
        KernelScope ks(ctx, "k_sort_gather");
        k_sort_gather<<<grid_of(ctx, n, SO_THREADS), SO_THREADS, 0, ctx->stream>>>(src, perm, 0, n, O, s->flags.as<int32_t>());
    }
    GSQL_CUDA(ctx, cudaGetLastError());
    h->rows = need;
    return GSQL_OK;
}

void held_init(Held *h, const gsql_sort_spec &spec) {
    h->rows = h->cap = 0;
    h->ncols = spec.n_cols;
    for (int e = 0; e < spec.n_cols; e++) {
        h->types[e] = spec.types[e];
        h->data[e].release();
        h->nulls[e].release();
        h->has_nulls[e] = false;
    }
}

// Cuts the held rows back to their best `limit`.
gsql_status held_cut(gsql_sort *s) {
    DevBuf perm;
    int64_t k = 0;
    const DColSet v = s->held.view();
    GSQL_TRY(topn_rows(s, v, s->held.rows, s->spec.limit, &perm, &k));
    Held *fresh = new Held();
    held_init(fresh, s->spec);
    gsql_status st = held_append(s, fresh, v, perm.as<uint32_t>(), k);
    if (st == GSQL_OK) {
        for (int e = 0; e < s->held.ncols; e++) {
            for (DevBuf *a : {&s->held.data[e], &s->held.nulls[e]}) a->ctx = s->ctx;
            for (DevBuf *a : {&fresh->data[e], &fresh->nulls[e]}) a->ctx = s->ctx;
            std::swap(s->held.data[e].p, fresh->data[e].p);
            std::swap(s->held.data[e].bytes, fresh->data[e].bytes);
            std::swap(s->held.nulls[e].p, fresh->nulls[e].p);
            std::swap(s->held.nulls[e].bytes, fresh->nulls[e].bytes);
            s->held.has_nulls[e] = fresh->has_nulls[e];
        }
        s->held.rows = fresh->rows;
        s->held.cap = fresh->cap;
    }
    delete fresh;  // frees the old buffers, stream-ordered after the gather
    return st;
}

}  // namespace

extern "C" gsql_status gsql_sort_create(gsql_ctx *ctx, const gsql_sort_spec *spec, gsql_sort **out) {
    if (!ctx || !spec || !out) return GSQL_E_INVALID;
    *out = nullptr;
    if (ctx->sticky) return GSQL_E_CUDA;
    if (spec->n_cols < 1 || spec->n_cols > GSQL_MAX_COLS)
        return gsql_set_error(ctx, GSQL_E_INVALID, "n_cols %d: must be in [1, %d]", spec->n_cols, GSQL_MAX_COLS);
    for (int i = 0; i < spec->n_cols; i++) {
        const int t = spec->types[i];
        if (t == GSQL_T_DEC128) return gsql_set_error(ctx, GSQL_E_UNSUPPORTED, "column %d: DEC128 columns are not sorted on the GPU", i);
        if (t != GSQL_T_INT32 && t != GSQL_T_INT64 && t != GSQL_T_FP64) return gsql_set_error(ctx, GSQL_E_INVALID, "column %d: unknown type %d", i, t);
    }
    if (spec->nkeys < 1 || spec->nkeys > GSQL_MAX_KEYS)
        return gsql_set_error(ctx, GSQL_E_INVALID, "nkeys %d: must be in [1, %d]", spec->nkeys, GSQL_MAX_KEYS);
    for (int k = 0; k < spec->nkeys; k++) {
        if (spec->key_col[k] < 0 || spec->key_col[k] >= spec->n_cols)
            return gsql_set_error(ctx, GSQL_E_INVALID, "sort key %d: column %d out of range", k, spec->key_col[k]);
        if (spec->key_desc[k] != 0 && spec->key_desc[k] != 1)
            return gsql_set_error(ctx, GSQL_E_INVALID, "sort key %d: key_desc %d is neither 0 nor 1", k, spec->key_desc[k]);
    }
    if (spec->limit < -1) return gsql_set_error(ctx, GSQL_E_INVALID, "limit %lld < 0 (topSize must not be negative)", (long long)spec->limit);
    GSQL_CUDA(ctx, cudaSetDevice(ctx->device));
    gsql_sort *s = new gsql_sort();
    s->ctx = ctx;
    s->spec = *spec;
    s->topn = spec->limit >= 0 && spec->limit <= TOPN_MAX_LIMIT;
    held_init(&s->held, *spec);
    gsql_status st = s->mm.alloc(ctx, sizeof(MinMax));
    if (st == GSQL_OK) st = s->hist.alloc(ctx, NBINS * 4);
    if (st == GSQL_OK) st = s->state.alloc(ctx, sizeof(TopnState));
    if (st == GSQL_OK) st = s->cur.alloc(ctx, 16);
    if (st == GSQL_OK) st = s->flags.alloc(ctx, 16);
    if (st == GSQL_OK && cudaMemsetAsync(s->flags.p, 0, 16, ctx->stream) != cudaSuccess) st = GSQL_E_CUDA;
    if (st != GSQL_OK) {
        delete s;
        return st;
    }
    gsql_ctx_retain(ctx);
    *out = s;
    return GSQL_OK;
}

extern "C" void gsql_sort_destroy(gsql_sort *s) {
    if (!s) return;
    gsql_ctx *ctx = s->ctx;
    cudaSetDevice(ctx->device);
    delete s;
    if (!ctx->sticky) cudaStreamSynchronize(ctx->stream);
    gsql_ctx_release(ctx);
}

extern "C" gsql_status gsql_sort_consume(gsql_sort *s, const gsql_batch *batch) {
    if (!s || !batch) return GSQL_E_INVALID;
    gsql_ctx *ctx = s->ctx;
    if (ctx->sticky) return GSQL_E_CUDA;
    if (s->finished) return gsql_set_error(ctx, GSQL_E_STATE, "consume after finish");
    GSQL_TRY(validate_batch(ctx, batch, s->spec.n_cols, s->spec.types));
    if (batch->rows == 0 || s->spec.limit == 0) return GSQL_OK;
    if (!s->topn && s->held.rows + batch->rows > MAX_ROW_IDS)
        return gsql_set_error(ctx, GSQL_E_CAPACITY, "%lld rows to sort exceed the 32-bit row ids (%lld)", (long long)(s->held.rows + batch->rows),
                              (long long)MAX_ROW_IDS);
    GSQL_CUDA(ctx, cudaSetDevice(ctx->device));
    StagedBatch sb;
    GSQL_TRY(stage_batch(ctx, batch, &sb));
    if (!s->topn) {
        DColSet src;
        memset(&src, 0, sizeof(src));
        src.n = sb.ncols;
        for (int e = 0; e < sb.ncols; e++) src.c[e] = sb.cols[e];
        GSQL_TRY(held_append(s, &s->held, src, nullptr, batch->rows));
    } else {
        const int64_t L = s->spec.limit;
        for (int64_t lo = 0; lo < batch->rows; lo += TOPN_SLICE) {  // row ids are 32-bit: a larger batch is selected slice by slice
            const int64_t n = batch->rows - lo < TOPN_SLICE ? batch->rows - lo : TOPN_SLICE;
            DColSet src;
            memset(&src, 0, sizeof(src));
            src.n = sb.ncols;
            for (int e = 0; e < sb.ncols; e++) {
                const DCol &c = sb.cols[e];
                src.c[e] = DCol{reinterpret_cast<const char *>(c.data) + (size_t)lo * gsql_type_width(c.type), c.nulls ? c.nulls + lo : nullptr,
                                c.type, 0};
            }
            if (n <= L) {
                GSQL_TRY(held_append(s, &s->held, src, nullptr, n));
            } else {
                DevBuf perm;
                int64_t k = 0;
                GSQL_TRY(topn_rows(s, src, n, L, &perm, &k));
                GSQL_TRY(held_append(s, &s->held, src, perm.as<uint32_t>(), k));
            }
            if (s->held.rows > (2 * L > TOPN_HOLD_MIN ? 2 * L : TOPN_HOLD_MIN)) GSQL_TRY(held_cut(s));
        }
    }
    if (batch->mem == GSQL_MEM_HOST) GSQL_CUDA(ctx, cudaStreamSynchronize(ctx->stream));  // staged copies die with `sb`
    return GSQL_OK;
}

extern "C" gsql_status gsql_sort_finish(gsql_sort *s, int64_t *rows) {
    if (!s || !rows) return GSQL_E_INVALID;
    gsql_ctx *ctx = s->ctx;
    if (ctx->sticky) return GSQL_E_CUDA;
    if (s->finished) return gsql_set_error(ctx, GSQL_E_STATE, "finish called twice");
    GSQL_CUDA(ctx, cudaSetDevice(ctx->device));
    const DColSet v = s->held.view();
    if (s->spec.limit >= 0) {
        GSQL_TRY(topn_rows(s, v, s->held.rows, s->spec.limit, &s->perm, &s->out_rows));
    } else {
        GSQL_TRY(sort_rows(s, v, nullptr, s->held.rows, &s->perm));
        s->out_rows = s->held.rows;
    }
    GSQL_CUDA(ctx, cudaStreamSynchronize(ctx->stream));
    s->finished = true;
    s->cursor = 0;
    *rows = s->out_rows;
    return GSQL_OK;
}

extern "C" gsql_status gsql_sort_next(gsql_sort *s, gsql_batch *out, int64_t max_rows, int64_t *out_rows) {
    if (!s || !out || !out_rows) return GSQL_E_INVALID;
    gsql_ctx *ctx = s->ctx;
    if (ctx->sticky) return GSQL_E_CUDA;
    *out_rows = 0;
    if (!s->finished) return gsql_set_error(ctx, GSQL_E_STATE, "next before finish");
    if (max_rows < 0) return gsql_set_error(ctx, GSQL_E_INVALID, "max_rows %lld < 0", (long long)max_rows);
    GSQL_TRY(validate_batch(ctx, out, s->spec.n_cols, s->spec.types));
    const int64_t left = s->out_rows - s->cursor, n = left < max_rows ? left : max_rows;
    out->rows = 0;
    if (n == 0) return GSQL_OK;
    GSQL_CUDA(ctx, cudaSetDevice(ctx->device));
    GatherOut O;
    memset(&O, 0, sizeof(O));
    DevBuf odata[GSQL_MAX_COLS], onull[GSQL_MAX_COLS];
    for (int e = 0; e < s->spec.n_cols; e++) {
        if (out->mem == GSQL_MEM_DEVICE) {
            O.data[e] = out->cols[e].data;
            O.nulls[e] = out->cols[e].nulls;
        } else {
            GSQL_TRY(odata[e].alloc(ctx, (size_t)n * gsql_type_width(s->spec.types[e])));
            O.data[e] = odata[e].p;
            if (out->cols[e].nulls) {
                GSQL_TRY(onull[e].alloc(ctx, (size_t)n));
                O.nulls[e] = onull[e].as<uint8_t>();
            }
        }
    }
    {
        KernelScope ks(ctx, "k_sort_gather");
        k_sort_gather<<<grid_of(ctx, n, SO_THREADS), SO_THREADS, 0, ctx->stream>>>(s->held.view(), s->perm.as<uint32_t>(), s->cursor, n, O,
                                                                                 s->flags.as<int32_t>());
    }
    GSQL_CUDA(ctx, cudaGetLastError());
    int32_t hf[4];
    GSQL_CUDA(ctx, cudaMemcpyAsync(hf, s->flags.p, 16, cudaMemcpyDeviceToHost, ctx->stream));
    GSQL_CUDA(ctx, cudaStreamSynchronize(ctx->stream));
    if (hf[0]) {
        GSQL_CUDA(ctx, cudaMemsetAsync(s->flags.p, 0, 16, ctx->stream));
        return gsql_set_error(ctx, GSQL_E_INVALID, "a NULL had to be written into an output column without a nulls buffer");
    }
    if (out->mem == GSQL_MEM_HOST) {
        for (int e = 0; e < s->spec.n_cols; e++) {
            GSQL_CUDA(ctx, cudaMemcpyAsync(out->cols[e].data, O.data[e], (size_t)n * gsql_type_width(s->spec.types[e]), cudaMemcpyDeviceToHost,
                                           ctx->stream));
            if (out->cols[e].nulls) GSQL_CUDA(ctx, cudaMemcpyAsync(out->cols[e].nulls, O.nulls[e], (size_t)n, cudaMemcpyDeviceToHost, ctx->stream));
        }
        GSQL_CUDA(ctx, cudaStreamSynchronize(ctx->stream));
    }
    s->cursor += n;
    *out_rows = out->rows = n;
    return GSQL_OK;
}

// ------------------------------------------------------------------------------------------------ merge of sorted runs
// gsql_merge_* (MergeSortExec / MergeSortedChunks.mergeSortedPages).  Batches are appended to one Held in arrival order
// with a host-side segment table.  finish() lists the held rows input by input (run_order, so run i is one contiguous
// range), plans the key images over all of them at once (one plan: images of different runs compare), and then:
//   * no group (every key constant): the output is run_order;
//   * one group of <= 128 bits: the images are encoded through run_order and the runs merged pairwise, ceil(log2 k)
//     rounds of a merge-path merge (k_merge_partition: one diagonal search per output tile; k_merge_tiles: a CTA stages
//     its two slices in shared memory, each thread merges MG_IPT items in registers, stores are coalesced).  Ties take
//     the left run, so the merge is stable.  With a limit each pair's output stops at L;
//   * more than one group: the stable radix sort of run_order, which orders rows exactly as the stable merge does.
// The tile kernel also checks that the slices it stages are ordered; a run that is not (its partitions need not be
// consistent then, and are clamped so that every access stays inside the run) sends the rows to the stable sort instead.
namespace {

constexpr int MG_THREADS = 128;
template <typename K> struct MergeIpt;  // items per thread: odd, so the register -> shared stores are conflict-free
template <> struct MergeIpt<uint32_t> { static constexpr int v = 15; };
template <> struct MergeIpt<uint64_t> { static constexpr int v = 11; };
template <> struct MergeIpt<K128> { static constexpr int v = 7; };

__device__ __forceinline__ bool key_less(uint32_t a, uint32_t b) { return a < b; }
__device__ __forceinline__ bool key_less(uint64_t a, uint64_t b) { return a < b; }
__device__ __forceinline__ bool key_less(const K128 &a, const K128 &b) { return a.hi < b.hi || (a.hi == b.hi && a.lo < b.lo); }

struct MergeSeg {  // held rows [src, src + rows) become run_order[dst, dst + rows)
    uint32_t src, dst, rows, pad;
};

// run_order[i] = held row of position i when the segments are laid out input by input (segments sorted by dst).
__global__ void __launch_bounds__(SO_THREADS) k_merge_run_order(const MergeSeg *__restrict__ segs, int nseg, int64_t n, uint32_t *__restrict__ out) {
    for (int64_t i = blockIdx.x * (int64_t)blockDim.x + threadIdx.x; i < n; i += (int64_t)gridDim.x * blockDim.x) {
        int lo = 0, hi = nseg - 1;
        while (lo < hi) {
            const int mid = (lo + hi + 1) >> 1;
            if (segs[mid].dst <= (uint64_t)i) lo = mid;
            else hi = mid - 1;
        }
        out[i] = segs[lo].src + (uint32_t)(i - segs[lo].dst);
    }
}

struct MergePair {  // run A = [a, a + na) and run B = [b, b + nb) merge into [out, out + n_out), n_out <= na + nb
    int64_t a, na, b, nb, out, n_out;
    int64_t tile0;  // first tile of this pair in the round
    int64_t part0;  // first partition slot of this pair (tile0 + pair index: each pair has one slot more than tiles)
};

__device__ __forceinline__ int find_pair(const MergePair *pairs, int npairs, int64_t x, bool by_part) {
    int lo = 0, hi = npairs - 1;
    while (lo < hi) {
        const int mid = (lo + hi + 1) >> 1;
        if ((by_part ? pairs[mid].part0 : pairs[mid].tile0) <= x) lo = mid;
        else hi = mid - 1;
    }
    return lo;
}

// Number of A items among the first d outputs of the stable merge of sorted A and B (ties take A).  Stays within
// [max(0, d - nb), min(d, na)] whatever the data.
template <typename K>
__device__ __forceinline__ int64_t merge_path(const K *A, int64_t na, const K *B, int64_t nb, int64_t d) {
    int64_t lo = d > nb ? d - nb : 0, hi = d < na ? d : na;
    while (lo < hi) {
        const int64_t mid = (lo + hi) >> 1;
        if (!key_less(B[d - 1 - mid], A[mid])) lo = mid + 1;
        else hi = mid;
    }
    return lo;
}

// parts[part0 + t] = the A split of pair p's output diagonal min(t * tile, n_out), t = 0 .. tiles(p).
template <typename K>
__global__ void __launch_bounds__(MG_THREADS) k_merge_partition(const MergePair *__restrict__ pairs, int npairs, int64_t nslots,
                                                                const K *__restrict__ keys, int64_t *__restrict__ parts) {
    constexpr int64_t TILE = (int64_t)MG_THREADS * MergeIpt<K>::v;
    for (int64_t j = blockIdx.x * (int64_t)blockDim.x + threadIdx.x; j < nslots; j += (int64_t)gridDim.x * blockDim.x) {
        const MergePair P = pairs[find_pair(pairs, npairs, j, true)];
        const int64_t d = (j - P.part0) * TILE < P.n_out ? (j - P.part0) * TILE : P.n_out;
        parts[j] = merge_path(keys + P.a, P.na, keys + P.b, P.nb, d);
    }
}

// One output tile per CTA.  keys_out == nullptr: the last round, only the row ids are written.  bad[0] is raised when a
// staged slice is out of order or the partitions are inconsistent (an input was not sorted).
template <typename K>
__global__ void __launch_bounds__(MG_THREADS) k_merge_tiles(const MergePair *__restrict__ pairs, int npairs, const K *__restrict__ keys_in,
                                                            const uint32_t *__restrict__ vals_in, const int64_t *__restrict__ parts,
                                                            K *__restrict__ keys_out, uint32_t *__restrict__ vals_out, int32_t *__restrict__ bad) {
    constexpr int IPT = MergeIpt<K>::v, TILE = MG_THREADS * IPT;
    __shared__ K sk[TILE];
    __shared__ uint32_t sv[TILE];
    const int64_t g = blockIdx.x;
    const int p = find_pair(pairs, npairs, g, false);
    const MergePair P = pairs[p];
    const int64_t t = g - P.tile0, d0 = t * TILE, d1 = d0 + TILE < P.n_out ? d0 + TILE : P.n_out;
    const int total = (int)(d1 - d0);
    const int64_t a0 = parts[P.part0 + t], a1 = parts[P.part0 + t + 1], b0 = d0 - a0;
    const int64_t na_raw = a1 - a0;
    const int na = (int)(na_raw < 0 ? 0 : (na_raw > total ? total : na_raw)), nb = total - na;
    bool unordered = threadIdx.x == 0 && na_raw != na;
    const K *A = keys_in + P.a + a0, *B = keys_in + P.b + b0;
    for (int i = threadIdx.x; i < total; i += MG_THREADS) {
        if (i < na) {
            sk[i] = A[i];
            sv[i] = vals_in[P.a + a0 + i];
        } else {
            sk[i] = B[i - na];
            sv[i] = vals_in[P.b + b0 + i - na];
        }
    }
    __syncthreads();
    for (int i = threadIdx.x; i < total; i += MG_THREADS) {  // each slice ordered, and after the item that precedes it
        if (i == 0 && na > 0 && a0 > 0) unordered |= key_less(sk[0], A[-1]);
        else if (i == na && nb > 0 && b0 > 0) unordered |= key_less(sk[na], B[-1]);
        else if (i != 0 && i != na) unordered |= key_less(sk[i], sk[i - 1]);
    }
    if (unordered) bad[0] = 1;
    const int diag = threadIdx.x * IPT < total ? threadIdx.x * IPT : total;
    int lo = diag > nb ? diag - nb : 0, hi = diag < na ? diag : na;
    while (lo < hi) {
        const int mid = (lo + hi) >> 1;
        if (!key_less(sk[na + diag - 1 - mid], sk[mid])) lo = mid + 1;
        else hi = mid;
    }
    int ai = lo, bi = na + diag - lo;
    K rk[IPT];
    uint32_t rv[IPT];
#pragma unroll
    for (int i = 0; i < IPT; i++) {
        if (diag + i < total) {
            const bool take_a = bi >= total || (ai < na && !key_less(sk[bi], sk[ai]));
            const int src = take_a ? ai : bi;
            rk[i] = sk[src];
            rv[i] = sv[src];
            ai += take_a;
            bi += !take_a;
        }
    }
    __syncthreads();
#pragma unroll
    for (int i = 0; i < IPT; i++)
        if (diag + i < total) {
            sk[diag + i] = rk[i];
            sv[diag + i] = rv[i];
        }
    __syncthreads();
    for (int i = threadIdx.x; i < total; i += MG_THREADS) {
        if (keys_out) keys_out[P.out + d0 + i] = sk[i];
        vals_out[P.out + d0 + i] = sv[i];
    }
}

struct MergeRun {
    int64_t off, len;
};

// Moves src's allocation into dst.
void take_buf(DevBuf *dst, DevBuf *src) {
    dst->release();
    dst->ctx = src->ctx;
    dst->p = src->p;
    dst->bytes = src->bytes;
    src->p = nullptr;
    src->bytes = 0;
}

}  // namespace

struct gsql_merge {
    gsql_sort *core;  // a full sort handle: the held rows, the key plan, the stable sort, next()'s gather and cursor
    int32_t n_inputs;
    int64_t limit;
    std::vector<MergeSeg> segs;  // arrival order; src = first held row
    std::vector<int32_t> seg_input;
    std::vector<int64_t> taken;  // rows held per input (each at most `limit`)
    bool finished = false;
    DevBuf bad;
};

namespace {

// out = the row ids of `runs` (encoded images in k0 / row ids in v0, both n long) merged pairwise round by round; *out_n
// = min(rows, limit).  *unordered: an input was found out of order (out is then not a valid result).
template <typename K>
gsql_status merge_runs(gsql_merge *m, const GroupEnc &g, const uint32_t *run_order, int64_t n, std::vector<MergeRun> runs, DevBuf *out,
                       int64_t *out_n, bool *unordered) {
    gsql_sort *s = m->core;
    gsql_ctx *ctx = s->ctx;
    constexpr int64_t TILE = (int64_t)MG_THREADS * MergeIpt<K>::v;
    DevBuf kb[2], vb[2], pairs_d, parts;
    for (int i = 0; i < 2; i++) {
        GSQL_TRY(kb[i].alloc(ctx, (size_t)n * sizeof(K)));
        GSQL_TRY(vb[i].alloc(ctx, (size_t)n * 4));
    }
    {
        KernelScope ks(ctx, "k_sort_encode");
        k_sort_encode<K><<<grid_of(ctx, n, SO_THREADS), SO_THREADS, 0, ctx->stream>>>(g, run_order, n, kb[0].as<K>(), vb[0].as<uint32_t>());
    }
    GSQL_CUDA(ctx, cudaGetLastError());
    GSQL_CUDA(ctx, cudaMemsetAsync(m->bad.p, 0, 16, ctx->stream));
    int cur = 0;
    std::vector<MergePair> pairs;
    while (runs.size() > 1) {
        pairs.clear();
        std::vector<MergeRun> next;
        int64_t out_at = 0, tiles = 0;
        for (size_t r = 0; r < runs.size(); r += 2) {  // an odd run is carried through as a merge with an empty run
            MergePair P;
            P.a = runs[r].off;
            P.na = runs[r].len;
            P.b = r + 1 < runs.size() ? runs[r + 1].off : 0;
            P.nb = r + 1 < runs.size() ? runs[r + 1].len : 0;
            P.n_out = P.na + P.nb;
            if (m->limit >= 0 && P.n_out > m->limit) P.n_out = m->limit;
            P.out = out_at;
            P.tile0 = tiles;
            P.part0 = tiles + (int64_t)pairs.size();
            tiles += div_up(P.n_out, TILE);
            out_at += P.n_out;
            pairs.push_back(P);
            next.push_back(MergeRun{P.out, P.n_out});
        }
        const bool last = next.size() == 1;
        const int64_t nslots = tiles + (int64_t)pairs.size();
        GSQL_TRY(pairs_d.alloc(ctx, pairs.size() * sizeof(MergePair)));
        GSQL_TRY(parts.alloc(ctx, (size_t)nslots * 8));
        GSQL_CUDA(ctx, cudaMemcpyAsync(pairs_d.p, pairs.data(), pairs.size() * sizeof(MergePair), cudaMemcpyHostToDevice, ctx->stream));
        {
            KernelScope ks(ctx, "k_merge_partition");
            k_merge_partition<K><<<grid_of(ctx, nslots, MG_THREADS), MG_THREADS, 0, ctx->stream>>>(pairs_d.as<MergePair>(), (int)pairs.size(), nslots,
                                                                                                  kb[cur].as<K>(), parts.as<int64_t>());
        }
        GSQL_CUDA(ctx, cudaGetLastError());
        {
            KernelScope ks(ctx, "k_merge_tiles");
            k_merge_tiles<K><<<(unsigned)tiles, MG_THREADS, 0, ctx->stream>>>(pairs_d.as<MergePair>(), (int)pairs.size(), kb[cur].as<K>(),
                                                                            vb[cur].as<uint32_t>(), parts.as<int64_t>(),
                                                                            last ? nullptr : kb[cur ^ 1].as<K>(), vb[cur ^ 1].as<uint32_t>(),
                                                                            m->bad.as<int32_t>());
        }
        GSQL_CUDA(ctx, cudaGetLastError());
        cur ^= 1;
        runs.swap(next);
    }
    int32_t hb[4];
    GSQL_CUDA(ctx, cudaMemcpyAsync(hb, m->bad.p, 16, cudaMemcpyDeviceToHost, ctx->stream));
    GSQL_CUDA(ctx, cudaStreamSynchronize(ctx->stream));
    *unordered = hb[0] != 0;
    *out_n = runs[0].len;
    take_buf(out, &vb[cur]);
    return GSQL_OK;
}

gsql_status merge_order(gsql_merge *m) {
    gsql_sort *s = m->core;
    gsql_ctx *ctx = s->ctx;
    const int64_t n = s->held.rows;
    // run_order: every input's segments in arrival order, input by input
    std::vector<MergeSeg> lay;
    std::vector<MergeRun> runs;
    std::vector<std::vector<size_t>> of_input(m->n_inputs);
    for (size_t i = 0; i < m->segs.size(); i++) of_input[m->seg_input[i]].push_back(i);
    int64_t at = 0;
    for (int in = 0; in < m->n_inputs; in++) {
        const int64_t off = at;
        for (size_t i : of_input[in]) {
            MergeSeg sg = m->segs[i];
            sg.dst = (uint32_t)at;
            at += sg.rows;
            if (!lay.empty() && lay.back().src + lay.back().rows == sg.src) lay.back().rows += sg.rows;  // contiguous in held
            else lay.push_back(sg);
        }
        if (at > off) runs.push_back(MergeRun{off, at - off});
    }
    DevBuf order, segs_d;
    GSQL_TRY(order.alloc(ctx, (size_t)n * 4));
    const int64_t want = m->limit >= 0 && m->limit < n ? m->limit : n;
    if (n == 0) {
        take_buf(&s->perm, &order);
        s->out_rows = 0;
        return GSQL_OK;
    }
    GSQL_TRY(segs_d.alloc(ctx, lay.size() * sizeof(MergeSeg)));
    GSQL_CUDA(ctx, cudaMemcpyAsync(segs_d.p, lay.data(), lay.size() * sizeof(MergeSeg), cudaMemcpyHostToDevice, ctx->stream));
    {
        KernelScope ks(ctx, "k_merge_run_order");
        k_merge_run_order<<<grid_of(ctx, n, SO_THREADS), SO_THREADS, 0, ctx->stream>>>(segs_d.as<MergeSeg>(), (int)lay.size(), n,
                                                                                     order.as<uint32_t>());
    }
    GSQL_CUDA(ctx, cudaGetLastError());
    s->out_rows = want;
    if (runs.size() <= 1) {  // one run: already in order
        take_buf(&s->perm, &order);
        return GSQL_OK;
    }
    const DColSet v = s->held.view();
    std::vector<GroupEnc> groups;
    GSQL_TRY(plan_groups(s, v, order.as<uint32_t>(), n, &groups));
    if (groups.empty()) {  // every key is constant: input by input is the stable order
        take_buf(&s->perm, &order);
        return GSQL_OK;
    }
    if (groups.size() == 1) {
        const GroupEnc &g = groups[0];
        bool unordered = false;
        int64_t got = 0;
        if (g.bits > 64) GSQL_TRY(merge_runs<K128>(m, g, order.as<uint32_t>(), n, runs, &s->perm, &got, &unordered));
        else if (g.bits > 32) GSQL_TRY(merge_runs<uint64_t>(m, g, order.as<uint32_t>(), n, runs, &s->perm, &got, &unordered));
        else GSQL_TRY(merge_runs<uint32_t>(m, g, order.as<uint32_t>(), n, runs, &s->perm, &got, &unordered));
        if (!unordered) {
            if (got != want) return gsql_set_error(ctx, GSQL_E_CUDA, "merge produced %lld rows, expected %lld", (long long)got, (long long)want);
            return GSQL_OK;
        }
    }
    // images over 128 bits, or an input out of order: the stable sort of the runs laid out input by input
    return sort_rows(s, v, order.as<uint32_t>(), n, &s->perm);
}

}  // namespace

extern "C" gsql_status gsql_merge_create(gsql_ctx *ctx, const gsql_sort_spec *spec, int32_t n_inputs, gsql_merge **out) {
    if (!ctx || !spec || !out) return GSQL_E_INVALID;
    *out = nullptr;
    if (ctx->sticky) return GSQL_E_CUDA;
    if (n_inputs < 1 || n_inputs > GSQL_MAX_MERGE_INPUTS)
        return gsql_set_error(ctx, GSQL_E_INVALID, "n_inputs %d: must be in [1, %d]", n_inputs, GSQL_MAX_MERGE_INPUTS);
    if (spec->limit < -1) return gsql_set_error(ctx, GSQL_E_INVALID, "limit %lld < 0", (long long)spec->limit);
    gsql_sort_spec full = *spec;
    full.limit = -1;  // the core holds every row it is given; the quota is applied here
    gsql_sort *core = nullptr;
    GSQL_TRY(gsql_sort_create(ctx, &full, &core));
    gsql_merge *m = new gsql_merge();
    m->core = core;
    m->n_inputs = n_inputs;
    m->limit = spec->limit;
    m->taken.assign(n_inputs, 0);
    const gsql_status st = m->bad.alloc(ctx, 16);
    if (st != GSQL_OK) {
        delete m;  // frees `bad` while the core still holds the context
        gsql_sort_destroy(core);
        return st;
    }
    *out = m;
    return GSQL_OK;
}

extern "C" void gsql_merge_destroy(gsql_merge *m) {
    if (!m) return;
    cudaSetDevice(m->core->ctx->device);
    m->bad.release();
    gsql_sort_destroy(m->core);
    delete m;
}

extern "C" gsql_status gsql_merge_consume(gsql_merge *m, int32_t input, const gsql_batch *batch) {
    if (!m || !batch) return GSQL_E_INVALID;
    gsql_sort *s = m->core;
    gsql_ctx *ctx = s->ctx;
    if (ctx->sticky) return GSQL_E_CUDA;
    if (m->finished) return gsql_set_error(ctx, GSQL_E_STATE, "consume after finish");
    if (input < 0 || input >= m->n_inputs) return gsql_set_error(ctx, GSQL_E_INVALID, "input %d: must be in [0, %d)", input, m->n_inputs);
    GSQL_TRY(validate_batch(ctx, batch, s->spec.n_cols, s->spec.types));
    int64_t n = batch->rows;
    if (m->limit >= 0 && n > m->limit - m->taken[input]) n = m->limit - m->taken[input];  // rows past the input's quota
    if (n <= 0) return GSQL_OK;
    if (s->held.rows + n > MAX_ROW_IDS)
        return gsql_set_error(ctx, GSQL_E_CAPACITY, "%lld rows to merge exceed the 32-bit row ids (%lld)", (long long)(s->held.rows + n),
                              (long long)MAX_ROW_IDS);
    GSQL_CUDA(ctx, cudaSetDevice(ctx->device));
    StagedBatch sb;
    GSQL_TRY(stage_batch(ctx, batch, &sb));
    DColSet src;
    memset(&src, 0, sizeof(src));
    src.n = sb.ncols;
    for (int e = 0; e < sb.ncols; e++) src.c[e] = sb.cols[e];
    const int64_t first = s->held.rows;
    GSQL_TRY(held_append(s, &s->held, src, nullptr, n));
    m->segs.push_back(MergeSeg{(uint32_t)first, 0, (uint32_t)n, 0});
    m->seg_input.push_back(input);
    m->taken[input] += n;
    if (batch->mem == GSQL_MEM_HOST) GSQL_CUDA(ctx, cudaStreamSynchronize(ctx->stream));  // staged copies die with `sb`
    return GSQL_OK;
}

extern "C" gsql_status gsql_merge_finish(gsql_merge *m, int64_t *rows) {
    if (!m || !rows) return GSQL_E_INVALID;
    gsql_sort *s = m->core;
    gsql_ctx *ctx = s->ctx;
    if (ctx->sticky) return GSQL_E_CUDA;
    if (m->finished) return gsql_set_error(ctx, GSQL_E_STATE, "finish called twice");
    GSQL_CUDA(ctx, cudaSetDevice(ctx->device));
    GSQL_TRY(merge_order(m));
    GSQL_CUDA(ctx, cudaStreamSynchronize(ctx->stream));
    m->finished = s->finished = true;
    s->cursor = 0;
    *rows = s->out_rows;
    return GSQL_OK;
}

extern "C" gsql_status gsql_merge_next(gsql_merge *m, gsql_batch *out, int64_t max_rows, int64_t *out_rows) {
    if (!m) return GSQL_E_INVALID;
    return gsql_sort_next(m->core, out, max_rows, out_rows);
}

#include "smj.cuh"  // SortMergeJoinExec: holds its inner rows in a gsql_sort core
