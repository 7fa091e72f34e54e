// join_fast.cuh — radix-partitioned, L2-resident hash join for a single integer equi-key (the C2 / TPC-H shape).
//
// Why: a random 16-byte table read is several times slower when the table lives in HBM (each one drags a whole-line
// fetch) than when the touched slice of the table fits the L2 (50 MB on H100; tools/microbench.cu measures both).  So for tables
// beyond L2 both sides are range-partitioned on the TABLE SLOT (slot = mulhi(key_hash, nslots), partition = the same
// hash's high bits scaled to P, i.e. partition p owns the contiguous slot range p; for dense build keys the direct
// table of KeyMap below, collision-free, partition = the slot's top lg P bits), rows are packed into fixed-stride
// 8-byte-word rows {key, payload...}, and build and probe walk partition after partition so that the active 16 MB
// slice of the table stays L2-resident while the rows stream through with evict-first loads/stores:
//     k_fj_hist        keys only          ->  [partition][block] histogram (build side, and probe batches that
//                                             cannot take the one-pass regions)
//     k_fj_scatter_sm  all columns        ->  packed rows in partition order (one 1024-thread CTA per SM, whole-SM tiles
//                                             brought in by bulk copies, shared-memory staged, 16-byte run writes).
//                                             Probe side: one pass into fixed per-partition regions, space reserved in blocks
//     k_fj_region_tail unused region rows ->  KEY_EMPTY
//     k_fj_build_split packed build rows  ->  rows grouped by slot block (2^lgB slots, one CTA's shared memory)
//     k_fj_build_slab  grouped rows       ->  table; each block built in shared memory, written once with full lines
//     k_fj_insert      deferred rows      ->  table (the few rows the two build kernels could not place)
//     k_fj_probe       packed probe rows  ->  output columns (one table read per probe row, warp-ballot compaction,
//                                             one global cursor bump per 2048-row tile, full-line column flush)
// Tables that fit L2 skip the partitioning: k_fj_table_init + k_fj_insert build them and k_fj_probe reads the probe rows
// straight from the input columns.
// The hash table holds whole build rows inline (stride = key + payload words), so a probe is ONE L2 access; the direct
// table (KeyMap below) holds no keys: BP = W - 1 payload words per slot plus an occupancy bitmap.  Duplicate build
// keys, NULLs, composite/double keys, non-equi conditions and outer-build joins take the generic path in join.cu
// (same results, two-pass sizing).
//
// Reference behaviour preserved: AbstractBufferedJoinExec.nextRows:185-264 for INNER / LEFT / RIGHT / SEMI / ANTI
// with unique build keys and no NULLs (row multiset identical; output order is unspecified in both).
#pragma once

#include <cub/block/block_scan.cuh>
#include <cub/device/device_scan.cuh>

#include "common.cuh"

namespace fj {

constexpr unsigned long long KEY_EMPTY = 0x8000000000000000ULL;
constexpr int THREADS = 512;           // 16 warps per CTA: two CTAs per SM give 32 resident warps at ~60 registers
constexpr int RPT = 4;                 // rows per thread per tile
constexpr int TILE = THREADS * RPT;    // 2048 rows
constexpr int MAX_WORDS = 4;           // packed row = key word + up to 3 payload words
constexpr int MAX_P = 1024;
constexpr int MAX_DISP = 4096;         // insert gives up (generic path) beyond this displacement
// FL_SPILL: a one-pass probe partition could not use its regions (a region overflowed, or a key equals KEY_EMPTY);
// the probe of that layout returns at once and the host re-runs the batch on the exact layout.
enum { FL_SENTINEL = 0, FL_DUP = 1, FL_DISP = 2, FL_NULLOUT = 3, FL_SPILL = 4, FL_COUNT = 5 };

struct Layout {
    int32_t nwords, ncols, key_col, key_i32;
    int32_t word[GSQL_MAX_COLS];
    int32_t half[GSQL_MAX_COLS];  // 0 = low 32 bits, 1 = high 32 bits, 2 = whole word
};

// Returns false when the side does not fit the packed-row format.
static bool make_layout(const int32_t *types, int ncols, int key_col, Layout *L) {
    memset(L, 0, sizeof(*L));
    L->ncols = ncols;
    L->key_col = key_col;
    L->key_i32 = types[key_col] == GSQL_T_INT32;
    int next = 1;
    int open_word = -1;  // a word whose high half is still free
    for (int c = 0; c < ncols; c++) {
        if (c == key_col) {
            L->word[c] = 0;
            L->half[c] = L->key_i32 ? 0 : 2;  // an INT32 key is stored widened; its low half is the column value
            continue;
        }
        if (types[c] == GSQL_T_INT32) {
            if (open_word >= 0) {
                L->word[c] = open_word;
                L->half[c] = 1;
                open_word = -1;
            } else {
                L->word[c] = next;
                L->half[c] = 0;
                open_word = next++;
            }
        } else {
            L->word[c] = next++;
            L->half[c] = 2;
        }
    }
    L->nwords = next;
    return next <= MAX_WORDS;
}

// Fibonacci (multiplicative) hashing: the well-mixed HIGH bits of key * phi64 are exactly what the mulhi range
// reductions (slot = mulhi(h, nslots), partition = mulhi(h, P)) consume; one 64-bit multiply instead of fmix64's two.
__device__ __forceinline__ uint64_t key_hash(unsigned long long k) { return (k ^ (k >> 32)) * 0x9E3779B97F4A7C15ULL; }

// Packs the RPT rows a thread owns in a tile (rows base + k*THREADS).  With a compile-time column count NC every load
// of the tile (NC x RPT coalesced loads) is issued before the first one is consumed; NC = 0 is the generic fallback
// (column loop not unrolled: RPT loads in flight per column).
template <int W, int NC>
__device__ __forceinline__ void pack_tile_nc(const DColSet &cols, const Layout &L, int64_t base, int64_t limit, unsigned long long (&w)[RPT][W]) {
    unsigned long long v[NC > 0 ? NC : 1][RPT];
#pragma unroll
    for (int c = 0; c < NC; c++) {
        const DCol &col = cols.c[c];
        const bool is32 = col.type == GSQL_T_INT32;
#pragma unroll
        for (int k = 0; k < RPT; k++) {
            int64_t r = base + k * THREADS;
            v[c][k] = 0;
            if (r < limit) {
                if (is32) v[c][k] = (unsigned long long)(unsigned)ld_stream_4(reinterpret_cast<const int *>(col.data) + r);
                else v[c][k] = (unsigned long long)ld_stream_8(reinterpret_cast<const long long *>(col.data) + r);
            }
        }
    }
#pragma unroll
    for (int k = 0; k < RPT; k++)
#pragma unroll
        for (int i = 0; i < W; i++) w[k][i] = 0;
#pragma unroll
    for (int c = 0; c < NC; c++) {
        const bool sext = c == L.key_col && cols.c[c].type == GSQL_T_INT32;
        const int wi = L.word[c];
        const int sh = L.half[c] == 1 ? 32 : 0;
#pragma unroll
        for (int k = 0; k < RPT; k++) {
            unsigned long long vv = sext ? (unsigned long long)(long long)(int)(unsigned)v[c][k] : v[c][k];
            vv <<= sh;
#pragma unroll
            for (int i = 0; i < W; i++)
                if (i == wi) w[k][i] |= vv;
        }
    }
}

template <int W>
__device__ __forceinline__ void pack_tile_generic(const DColSet &cols, const Layout &L, int64_t base, int64_t limit, unsigned long long (&w)[RPT][W]) {
#pragma unroll
    for (int k = 0; k < RPT; k++)
#pragma unroll
        for (int i = 0; i < W; i++) w[k][i] = 0;
#pragma unroll 1
    for (int c = 0; c < L.ncols; c++) {
        const DCol &col = cols.c[c];
        const bool is32 = col.type == GSQL_T_INT32, iskey = c == L.key_col;
        const int wi = L.word[c];
        const int sh = L.half[c] == 1 ? 32 : 0;
        unsigned long long v[RPT];
#pragma unroll
        for (int k = 0; k < RPT; k++) {
            int64_t r = base + k * THREADS;
            v[k] = 0;
            if (r < limit) {
                if (is32) {
                    int x = ld_stream_4(reinterpret_cast<const int *>(col.data) + r);
                    v[k] = iskey ? (unsigned long long)(long long)x : (unsigned long long)(unsigned)x;
                } else {
                    v[k] = (unsigned long long)ld_stream_8(reinterpret_cast<const long long *>(col.data) + r);
                }
            }
        }
#pragma unroll
        for (int k = 0; k < RPT; k++) {
            unsigned long long vv = v[k] << sh;
#pragma unroll
            for (int i = 0; i < W; i++)
                if (i == wi) w[k][i] |= vv;
        }
    }
}

template <int W>
__device__ __forceinline__ void pack_tile(const DColSet &cols, const Layout &L, int64_t base, int64_t limit, unsigned long long (&w)[RPT][W]) {
    switch (L.ncols) {  // warp-uniform
    case 1: pack_tile_nc<W, 1>(cols, L, base, limit, w); break;
    case 2: pack_tile_nc<W, 2>(cols, L, base, limit, w); break;
    case 3: pack_tile_nc<W, 3>(cols, L, base, limit, w); break;
    case 4: pack_tile_nc<W, 4>(cols, L, base, limit, w); break;
    default: pack_tile_generic<W>(cols, L, base, limit, w); break;
    }
}

__device__ __forceinline__ unsigned long long load_key(const DCol &col, int64_t r) {
    if (col.type == GSQL_T_INT32) return (unsigned long long)(long long)ld_stream_4(reinterpret_cast<const int *>(col.data) + r);
    return (unsigned long long)ld_stream_8(reinterpret_cast<const long long *>(col.data) + r);
}

// Partition of a key hash.  Only the high 32 bits take part (one IMAD.HI): the result may differ from
// slot / slots_per_partition for a vanishing fraction of keys, which costs those rows an access outside the resident
// slice, never correctness (slots are always addressed globally).
__device__ __forceinline__ unsigned int part_of(uint64_t h, int P) { return __umulhi((unsigned int)(h >> 32), (unsigned int)P); }

// The direct table, for build keys whose range is compact: with d = key - kmin and 2^bits slots,
// slot = (d * phi64) mod 2^bits.  Multiplying by an odd constant is a bijection on [0, 2^bits), so distinct build keys
// never share a slot.  A probe key k matches exactly when d = k - kmin (unsigned) is below 2^bits and a build row
// occupies slot(d), so the table stores no keys: slot s holds the build row's BP = W - 1 payload words at
// table[s * BP], and bit s of the occupancy bitmap that follows the payload (nslots bits, 32-bit words; a key-only
// build side has the bitmap alone) is set.  No key value is reserved, KEY_EMPTY included.  Partition p is the slot
// range whose top lgP bits are p; the multiply spreads clustered and strided key sets evenly over the partitions.  The
// kernels take the mode as a template parameter DIRECT; the hash mode (slot = mulhi(key_hash, nslots), linear
// probing) ignores M.
// When the build keys are exactly [kmin, kmin + dense) (dense > 0: as many distinct keys as values in their range, the
// shape of surrogate keys), every slot of that range is occupied, and the probe's range test d < dense replaces the
// bitmap read.
struct KeyMap {
    unsigned long long kmin;
    unsigned long long dense;
    int32_t bits, lgP;
};

// Bytes of the direct table for W-word build rows (payload words, then the bitmap; nslots >= 1024 is a power of two).
__host__ __device__ constexpr size_t direct_table_bytes(int W, uint64_t nslots) { return (size_t)nslots * (W - 1) * 8 + nslots / 8; }

template <int W>
__device__ __forceinline__ unsigned int *direct_bitmap(unsigned long long *table, uint64_t nslots) {
    return reinterpret_cast<unsigned int *>(table + nslots * (W - 1));
}
template <int W>
__device__ __forceinline__ const unsigned int *direct_bitmap(const unsigned long long *table, uint64_t nslots) {
    return reinterpret_cast<const unsigned int *>(table + nslots * (W - 1));
}

template <bool DIRECT>
__device__ __forceinline__ uint64_t slot_of(unsigned long long k, uint64_t nslots, const KeyMap &M) {
    if (DIRECT) return ((k - M.kmin) * 0x9E3779B97F4A7C15ULL) & (nslots - 1);
    return __umul64hi(key_hash(k), nslots);
}

template <bool DIRECT>
__device__ __forceinline__ unsigned int part_of_key(unsigned long long k, int P, const KeyMap &M) {
    if (DIRECT) return (unsigned int)(slot_of<true>(k, 1ULL << M.bits, M) >> (M.bits - M.lgP));
    return part_of(key_hash(k), P);
}

// Smallest and largest key of a column (signed): out[0] = min, out[1] = max, set to INT64_MAX / INT64_MIN beforehand.
__global__ void __launch_bounds__(256) k_fj_key_range(DCol keycol, int64_t n, long long *out) {
    constexpr int U = 4;  // loads in flight per thread
    long long lo = LLONG_MAX, hi = LLONG_MIN;
    const int64_t stride = (int64_t)gridDim.x * blockDim.x;
    for (int64_t r = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; r < n; r += U * stride) {
        long long k[U];
#pragma unroll
        for (int u = 0; u < U; u++) k[u] = r + u * stride < n ? (long long)load_key(keycol, r + u * stride) : 0;
#pragma unroll
        for (int u = 0; u < U; u++) {
            if (r + u * stride >= n) continue;
            lo = k[u] < lo ? k[u] : lo;
            hi = k[u] > hi ? k[u] : hi;
        }
    }
#pragma unroll
    for (int d = 16; d > 0; d >>= 1) {
        const long long a = __shfl_xor_sync(0xffffffffu, lo, d), b = __shfl_xor_sync(0xffffffffu, hi, d);
        lo = a < lo ? a : lo;
        hi = b > hi ? b : hi;
    }
    if ((threadIdx.x & 31) == 0 && lo <= hi) {
        atomicMin(out, lo);
        atomicMax(out + 1, hi);
    }
}

struct PartGeom {
    int64_t rows, chunk;  // rows per block (multiple of TILE)
    int32_t P, nblocks;
};

// ---- pass 1: histogram of partition ids, keys only.  It runs on the scatter's geometry (one histogram column per
// scatter block, one 1024-thread CTA per SM), so each CTA keeps as many loads in flight per SM as two 512-thread blocks do.
constexpr int SM_THREADS = 1024;

template <bool DIRECT>
__global__ void __launch_bounds__(SM_THREADS) k_fj_hist(DCol keycol, PartGeom g, int64_t *__restrict__ hist, int32_t *flags, KeyMap M) {
    extern __shared__ unsigned int sh_hist[];
    for (int i = threadIdx.x; i < g.P; i += SM_THREADS) sh_hist[i] = 0;
    __syncthreads();
    int64_t r0 = (int64_t)blockIdx.x * g.chunk;
    int64_t r1 = r0 + g.chunk < g.rows ? r0 + g.chunk : g.rows;
    bool sentinel = false;
    for (int64_t t0 = r0; t0 < r1; t0 += SM_THREADS * RPT) {
        unsigned long long key[RPT];
#pragma unroll
        for (int k = 0; k < RPT; k++) {
            int64_t r = t0 + k * SM_THREADS + threadIdx.x;
            key[k] = r < r1 ? load_key(keycol, r) : 0;
        }
#pragma unroll
        for (int k = 0; k < RPT; k++) {
            int64_t r = t0 + k * SM_THREADS + threadIdx.x;
            if (r < r1) {
                sentinel |= key[k] == KEY_EMPTY;
                atomicAdd(&sh_hist[part_of_key<DIRECT>(key[k], g.P, M)], 1u);
            }
        }
    }
    if (!DIRECT && sentinel) flags[FL_SENTINEL] = 1;  // the hash table's empty marker; the direct table has none
    __syncthreads();
    for (int i = threadIdx.x; i < g.P; i += SM_THREADS) hist[(int64_t)i * g.nblocks + blockIdx.x] = sh_hist[i];
}

// ---- pass 2: pack rows and scatter them into partition order through a shared-memory staged tile, one 1024-thread CTA
// per SM and one large tile per CTA.  A 2048-row tile gives each of C2's ~290 partitions ~7 rows (~114 B): less than a 128-byte line,
// so successive tiles write most lines in pieces, and the scatter ran at ~60 % of the streaming rate.  Here the tile is
// SM_THREADS * rpt rows, with rpt (<= sm_rpt_max(W)) chosen on the host as the largest that the SM's shared memory
// holds (6144 rows for W = 2 and P ~ 300: ~21 rows per partition run).  There is one input buffer: each column of a full
// tile arrives by one bulk copy (cp.async.bulk, issued by lane 0 of warp c for column c, completion on one mbarrier);
// columns whose base is not 16-byte aligned, and all columns of the ragged last tile, are loaded with per-thread
// cp.async into the same layout.  Once every thread holds its rows in registers (barrier A) the next tile's copies are
// started, so they overlap the scan, staging and flush of the current tile.  For 16-byte rows (W == 2) a run whose end
// falls inside a 32-byte sector holds its last row back: the row is restaged at the front of the partition's run in
// the CTA's next tile (its destination is the row just before that run's), so the same warp store writes the whole
// sector.  A sector written in two halves, a tile apart, costs far more HBM time than a whole one (DESIGN.md §4).
__host__ __device__ constexpr int sm_rpt_max(int W) { return W == 1 ? 8 : W == 2 ? 6 : W == 3 ? 4 : 3; }  // rows in registers: <= 12 words

// W == 2 (16-byte rows) carries a run's odd last row to the partition's next run, so that every flushed run ends on a
// 32-byte sector: the stage and spid hold up to P carried rows more, plus a P-row carry buffer and P hold indices.
__host__ __device__ constexpr bool sm_carry(int W) { return W == 2; }

static size_t scatter_sm_smem_bytes(int W, int P, int rpt) {
    const size_t T = (size_t)SM_THREADS * rpt, TS = T + (sm_carry(W) ? P : 0);
    // stage + input buffer, cur/delta/delta2/hist/start/split, spid, carry buffer + hold
    return TS * W * 8 + T * W * 8 + (size_t)P * (8 * 3 + 4 * 3) + TS * 2 + (sm_carry(W) ? (size_t)P * (W * 8 + 4) : 0);
}

// One-pass layout of the probe side: partition p owns rows [p * cap, p * cap + cap) of the packed buffer.  A CTA takes
// space in a region K rows at a time (K a power of two dividing cap, so every block is K-aligned) with one atomicAdd on
// fill[p].  It always holds a current block and one reserved next block, so the atomic that replaces a consumed next
// block is only waited for a tile later.  K == 0 selects the exact layout (offsets from k_fj_hist and a scan).
struct Regions {
    unsigned long long *fill;  // P: rows of region p handed out so far
    int64_t cap;
    int32_t K;
};

template <int W, bool DIRECT>
__global__ void __launch_bounds__(SM_THREADS, 1) k_fj_scatter_sm(const __grid_constant__ DColSet cols, const __grid_constant__ Layout L, PartGeom g,
                                                                 int rpt, const int64_t *__restrict__ offs, Regions RG,
                                                                 unsigned long long *__restrict__ out, int32_t *flags, KeyMap M) {
    constexpr int R = sm_rpt_max(W);
    constexpr bool CARRY = sm_carry(W);
    const int T = SM_THREADS * rpt, TS = T + (CARRY ? g.P : 0);
    extern __shared__ __align__(128) unsigned char smem_raw[];
    unsigned long long *stage = reinterpret_cast<unsigned long long *>(smem_raw);       // TS * W
    unsigned char *inbuf = reinterpret_cast<unsigned char *>(stage + (size_t)TS * W);   // column c at T * (bytes of columns < c)
    // CARRY: P * W, the held-back row of p (16-byte accesses: it follows the 16-byte-multiple stage and input buffer)
    unsigned long long *carry = reinterpret_cast<unsigned long long *>(inbuf + (size_t)T * W * 8);
    unsigned long long *cur = carry + (CARRY ? (size_t)g.P * W : 0);                    // P
    unsigned long long *delta = cur + g.P;                                              // P: destination - stage index, rows < split
    unsigned long long *delta2 = delta + g.P;                                           // P: the same for rows >= split
    unsigned int *hist = reinterpret_cast<unsigned int *>(delta2 + g.P);                // P
    unsigned int *start = hist + g.P;                                                   // P: stage index of p's first new row
    unsigned int *split = start + g.P;                                                  // P: first stage index in the next block
    unsigned int *hold = split + g.P;                                                   // CARRY: P, stage index of the row to hold back
    unsigned short *spid = reinterpret_cast<unsigned short *>(hold + (CARRY ? g.P : 0));  // TS
    __shared__ __align__(8) unsigned long long bar;
    __shared__ int spill;
    typedef cub::BlockScan<unsigned int, SM_THREADS, cub::BLOCK_SCAN_WARP_SCANS> BlockScan;
    __shared__ typename BlockScan::TempStorage scan_tmp;
    const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;

    // bytes of a full tile that arrive by bulk copy (uniform), and where column `warp` sits in the input buffer
    uint32_t bulk_bytes = 0, my_off = 0, off = 0;
    bool my_bulk = false;
    for (int c = 0; c < L.ncols; c++) {
        const uint32_t bytes = (uint32_t)T * (cols.c[c].type == GSQL_T_INT32 ? 4u : 8u);
        const bool aligned = ((uintptr_t)cols.c[c].data & 15) == 0;
        if (c == warp) { my_off = off; my_bulk = aligned; }
        off += bytes;
        if (aligned) bulk_bytes += bytes;
    }
    const bool issuer = lane == 0 && warp < L.ncols && my_bulk;
    uint64_t pol = 0;
    if (issuer) pol = l2_policy_evict_first();

    if (tid == 0) {
        mbar_init(&bar, 1);
        asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
        spill = 0;
    }
    static_assert(MAX_P <= SM_THREADS, "one partition per thread");
    const unsigned long long K = (unsigned long long)RG.K;
    unsigned long long nxt = 0;  // regions: thread p's reserved next block in region p (offset in the region)
    if (tid < g.P) {
        if (K) {
            const unsigned long long r = atomicAdd(&RG.fill[tid], 2 * K);
            if (r + 2 * K > (unsigned long long)RG.cap) spill = 1;
            cur[tid] = (unsigned long long)tid * RG.cap + r;
            nxt = r + K;
        } else {
            cur[tid] = (unsigned long long)offs[(int64_t)tid * g.nblocks + blockIdx.x];
        }
        hist[tid] = 0;
    }
    __syncthreads();
    if (spill) {
        if (tid == 0) flags[FL_SPILL] = 1;
        return;
    }
    const int64_t r0 = (int64_t)blockIdx.x * g.chunk;
    const int64_t r1 = r0 + g.chunk < g.rows ? r0 + g.chunk : g.rows;

    // starts the loads of the tile at t0 (n_tile rows) into inbuf
    auto load_tile = [&](int64_t t0, int n_tile) {
        const bool full = n_tile == T;
        if (full && bulk_bytes) {
            if (tid == 0) mbar_expect_tx(&bar, bulk_bytes);
            if (issuer) {
                const DCol &col = cols.c[warp];
                const uint32_t width = col.type == GSQL_T_INT32 ? 4u : 8u;
                tma_load_1d(inbuf + my_off, reinterpret_cast<const unsigned char *>(col.data) + t0 * width, (uint32_t)T * width, &bar, pol);
            }
        }
        unsigned char *sp = inbuf;
#pragma unroll 1
        for (int c = 0; c < L.ncols; c++) {
            const DCol &col = cols.c[c];
            const bool is32 = col.type == GSQL_T_INT32;
            if (!(full && ((uintptr_t)col.data & 15) == 0)) {
#pragma unroll
                for (int k = 0; k < R; k++) {
                    const int e = k * SM_THREADS + tid;
                    if (k < rpt && e < n_tile) {
                        if (is32) cp_async_4(sp + e * 4, reinterpret_cast<const int *>(col.data) + t0 + e);
                        else cp_async_8(sp + e * 8, reinterpret_cast<const long long *>(col.data) + t0 + e);
                    }
                }
            }
            sp += (size_t)T * (is32 ? 4 : 8);
        }
        cp_async_commit();
    };

    uint32_t phase = 0;
    unsigned int cc = 0;  // CARRY, thread p: rows of partition p held back by the previous tile (0 or 1)
    if (r0 < r1) load_tile(r0, (int)(r1 - r0 < T ? r1 - r0 : T));
    for (int64_t t0 = r0; t0 < r1; t0 += T) {
        const int n_tile = (int)(r1 - t0 < T ? r1 - t0 : T);
        // 1. wait for this tile's columns, pack this thread's rows (element k * SM_THREADS + tid) into registers
        if (n_tile == T && bulk_bytes) {
            mbar_wait(&bar, phase);
            phase ^= 1u;
        }
        cp_async_wait<0>();
        unsigned long long w[R][W];
#pragma unroll
        for (int k = 0; k < R; k++)
#pragma unroll
            for (int i = 0; i < W; i++) w[k][i] = 0;
        {
            const unsigned char *sp = inbuf;
#pragma unroll 1
            for (int c = 0; c < L.ncols; c++) {
                const bool is32 = cols.c[c].type == GSQL_T_INT32, iskey = c == L.key_col;
                const int wi = L.word[c];
                const int sh = L.half[c] == 1 ? 32 : 0;
#pragma unroll
                for (int k = 0; k < R; k++) {
                    const int e = k * SM_THREADS + tid;
                    if (k < rpt && e < n_tile) {
                        unsigned long long v;
                        if (is32) {
                            const int x = *reinterpret_cast<const int *>(sp + e * 4);
                            v = iskey ? (unsigned long long)(long long)x : (unsigned long long)(unsigned)x;
                        } else {
                            v = *reinterpret_cast<const unsigned long long *>(sp + e * 8);
                        }
#pragma unroll
                        for (int i = 0; i < W; i++)
                            if (i == wi) w[k][i] |= v << sh;
                    }
                }
                sp += (size_t)T * (is32 ? 4 : 8);
            }
        }
        // 2. rank: pid in the high half, rank within (tile, partition) in the low half (T <= 8192 rows, P <= 1024)
        unsigned int pr[R];
#pragma unroll
        for (int k = 0; k < R; k++) {
            pr[k] = 0xffffffffu;
            if (k < rpt && k * SM_THREADS + tid < n_tile) {
                const unsigned int pid = part_of_key<DIRECT>(w[k][0], g.P, M);
                pr[k] = (pid << 16) | atomicAdd(&hist[pid], 1u);
                if (K && w[k][0] == KEY_EMPTY) flags[FL_SPILL] = 1;  // a real key would read as a gap row
            }
        }
        __syncthreads();  // (A) every row of the tile is in registers and ranked: the input buffer can be refilled
        const bool more = t0 + T < r1;
        const int n_next = more ? (int)(r1 - (t0 + T) < T ? r1 - (t0 + T) : T) : 0;
        if (more) load_tile(t0 + T, n_next);
        unsigned int n_stage, my_start = 0;  // rows staged this tile (new + carried); thread p: start[p]
        {  // 3. exclusive scan of hist[0..P) (+ carried rows) -> start[]; delta[p] = (global cursor of p) - start[p]
            const int p = tid;
            unsigned int v = p < g.P ? hist[p] + cc : 0;
            BlockScan(scan_tmp).ExclusiveSum(v, v, n_stage);
            if (p < g.P) {
                v += cc;  // the carried row sits just before p's new rows, as its destination does
                my_start = v;
                start[p] = v;
                const unsigned int h = hist[p];
                const unsigned long long c = cur[p];
                delta[p] = c - v;
                split[p] = v + h;
                cur[p] = c + h;
                const unsigned int room = K ? (unsigned int)(K - (c & (K - 1))) : 0xffffffffu;
                if (h >= room) {  // the run fills the current block: its rest goes to the next block, or to a fresh
                                  // reservation of whole blocks when it does not fit one
                    const unsigned long long rest = h - room;
                    unsigned long long b, span = K;
                    if (rest < K) {
                        b = nxt;
                        nxt = atomicAdd(&RG.fill[p], K);  // first used at a later tile's scan
                    } else {
                        span = (rest / K + 1) * K;
                        b = atomicAdd(&RG.fill[p], span);
                    }
                    if (b + span > (unsigned long long)RG.cap) {  // the region is full: the host re-runs the exact path
                        spill = 1;
                        flags[FL_SPILL] = 1;
                    }
                    const unsigned long long base = (unsigned long long)p * RG.cap + b;
                    split[p] = v + room;
                    delta2[p] = base - (v + room);
                    cur[p] = base + rest;
                }
                if (CARRY) {  // a run that ends inside a 32-byte sector holds its last row back for the partition's next
                              // run (adjacent: with K >= 2 an odd end is inside a block), unless this is the last tile
                    const bool h_odd = more && K != 1 && (cur[p] & 1) && h + cc > 0;
                    hold[p] = h_odd ? v + h - 1 : 0xffffffffu;
                }
                hist[p] = 0;
            }
        }
        __syncthreads();  // (B)
        if (spill) {  // nothing more is written; the next tile's loads land before the CTA leaves
            if (more && n_next == T && bulk_bytes) mbar_wait(&bar, phase);
            cp_async_wait<0>();
            return;
        }
        // 4. stage the rows in partition order, each partition's carried row first
        if (CARRY && cc) {
            *reinterpret_cast<int4 *>(stage + (size_t)(my_start - 1) * 2) = *reinterpret_cast<const int4 *>(carry + (size_t)tid * 2);
            spid[my_start - 1] = (unsigned short)tid;
        }
        if (CARRY && tid < g.P) cc = hold[tid] != 0xffffffffu;
#pragma unroll
        for (int k = 0; k < R; k++) {
            if (pr[k] != 0xffffffffu) {
                const unsigned int pid = pr[k] >> 16;
                const unsigned int pos = start[pid] + (pr[k] & 0xffffu);
                if (W == 2) {
                    int4 v;
                    v.x = (int)(unsigned)w[k][0]; v.y = (int)(unsigned)(w[k][0] >> 32);
                    v.z = (int)(unsigned)w[k][W - 1]; v.w = (int)(unsigned)(w[k][W - 1] >> 32);
                    *reinterpret_cast<int4 *>(stage + (size_t)pos * 2) = v;
                } else {
#pragma unroll
                    for (int i = 0; i < W; i++) stage[(size_t)pos * W + i] = w[k][i];
                }
                spid[pos] = (unsigned short)pid;
            }
        }
        __syncthreads();  // (C)
        // 5. flush: consecutive threads -> consecutive addresses of a run.  No barrier after it: the next writes of
        // stage / spid / delta / carry come after the next tile's barrier (A), which every thread reaches only once its
        // flush is done.
#pragma unroll
        for (int k = 0; k < R + (CARRY ? 1 : 0); k++) {
            const int i = k * SM_THREADS + tid;
            if (i < (int)n_stage) {
                const unsigned int p = spid[i];
                const unsigned long long dst = ((unsigned)i < split[p] ? delta[p] : delta2[p]) + (unsigned)i;
                if (CARRY && (unsigned)i == hold[p]) {
                    *reinterpret_cast<int4 *>(carry + (size_t)p * 2) = *reinterpret_cast<const int4 *>(stage + (size_t)i * 2);
                } else if (W == 2) {
                    st_stream_16(out + dst * 2, *reinterpret_cast<const int4 *>(stage + (size_t)i * 2));
                } else {
#pragma unroll
                    for (int j = 0; j < W; j++) st_stream_8(out + dst * W + j, (long long)stage[(size_t)i * W + j]);
                }
            }
        }
    }
    if (K) {  // the unused rest of the current block and the unused next block of every partition become gap rows
        __syncthreads();  // every flush has read delta2
        if (tid < g.P) delta2[tid] = nxt;
        __syncthreads();
        for (int p = warp; p < g.P; p += SM_THREADS / 32) {
            const unsigned long long c = cur[p], e = (c | (K - 1)) + 1;
            const unsigned long long base = (unsigned long long)p * RG.cap, n0 = delta2[p];
            const unsigned long long n1 = n0 + K < (unsigned long long)RG.cap ? n0 + K : (unsigned long long)RG.cap;
            for (unsigned long long r = c + lane; r < e; r += 32) st_stream_8(out + r * W, (long long)KEY_EMPTY);
            for (unsigned long long r = base + n0 + lane; r < base + n1; r += 32) st_stream_8(out + r * W, (long long)KEY_EMPTY);
        }
    }
}

// One-pass layout: the rows of each region that no CTA reserved, [fill[p], cap), become gap rows.  One block per partition.
__global__ void __launch_bounds__(256) k_fj_region_tail(Regions RG, int W, unsigned long long *out) {
    const unsigned long long p = blockIdx.x, cap = (unsigned long long)RG.cap, f = RG.fill[p];
    for (unsigned long long r = p * cap + (f < cap ? f : cap) + threadIdx.x; r < (p + 1) * cap; r += 256)
        st_stream_8(out + r * W, (long long)KEY_EMPTY);
}

// ---- table
template <int W>
__global__ void __launch_bounds__(THREADS) k_fj_table_init(unsigned long long *table, uint64_t nslots) {
    for (uint64_t i = blockIdx.x * (uint64_t)blockDim.x + threadIdx.x; i < nslots; i += (uint64_t)gridDim.x * blockDim.x) {
        table[i * W] = KEY_EMPTY;
#pragma unroll
        for (int j = 1; j < W; j++) table[i * W + j] = 0;
    }
}

// Inserts rows (packed, or packed on the fly from columns when `packed` == nullptr).  Tiles are taken in index order
// so that concurrently running blocks work on neighbouring partitions (the table slice stays in L2).  `n_dev`, when
// given, holds a row count known only on the device (the slab build's deferred rows); n is then its upper bound.
// The direct table needs its bitmap cleared beforehand; the hash table, k_fj_table_init.
template <int W, bool DIRECT>
__global__ void __launch_bounds__(THREADS, 2) k_fj_insert(const unsigned long long *__restrict__ packed, const __grid_constant__ DColSet cols,
                                                       const __grid_constant__ Layout L, int64_t n, unsigned long long *table, uint64_t nslots,
                                                       int32_t *flags, const unsigned long long *n_dev, KeyMap M) {
    if (n_dev && *n_dev < (unsigned long long)n) n = (int64_t)*n_dev;
    for (int64_t t0 = (int64_t)blockIdx.x * TILE; t0 < n; t0 += (int64_t)gridDim.x * TILE) {
        unsigned long long w[RPT][W];
        if (packed) {
#pragma unroll
            for (int k = 0; k < RPT; k++) {
                int64_t r = t0 + k * THREADS + threadIdx.x;
#pragma unroll
                for (int i = 0; i < W; i++) w[k][i] = r < n ? (unsigned long long)ld_stream_8(packed + r * W + i) : 0;
            }
        } else {
            pack_tile<W>(cols, L, t0 + threadIdx.x, n, w);
        }
        if constexpr (DIRECT) {  // the row's own slot: set its bit, write its payload; a bit already set is a duplicate
            unsigned int *bm = direct_bitmap<W>(table, nslots);
#pragma unroll
            for (int k = 0; k < RPT; k++) {
                if (t0 + k * THREADS + threadIdx.x >= n) continue;
                const uint64_t s = slot_of<true>(w[k][0], nslots, M);
                const unsigned int bit = 1u << (s & 31);
                if (atomicOr(bm + (s >> 5), bit) & bit) {
                    flags[FL_DUP] = 1;
                    continue;
                }
#pragma unroll
                for (int i = 1; i < W; i++) table[s * (W - 1) + i - 1] = w[k][i];
            }
            continue;
        }
        // CAS attempts in rounds: every round issues one attempt for all still-unplaced rows of the thread
        uint64_t sl[RPT];
        unsigned long long prev[RPT];
        bool pending[RPT];
        bool any = false;
#pragma unroll
        for (int k = 0; k < RPT; k++) {
            int64_t r = t0 + k * THREADS + threadIdx.x;
            sl[k] = slot_of<DIRECT>(w[k][0], nslots, M);
            pending[k] = r < n;
            if (pending[k] && w[k][0] == KEY_EMPTY) { flags[FL_SENTINEL] = 1; pending[k] = false; }
            any |= pending[k];
        }
        int disp = 0;
        while (__any_sync(0xffffffffu, any)) {
#pragma unroll
            for (int k = 0; k < RPT; k++)
                if (pending[k]) prev[k] = atomicCAS(table + sl[k] * W, KEY_EMPTY, w[k][0]);
            any = false;
#pragma unroll
            for (int k = 0; k < RPT; k++) {
                if (!pending[k]) continue;
                if (prev[k] == KEY_EMPTY) {  // claimed: the payload words follow (visible after the kernel)
#pragma unroll
                    for (int i = 1; i < W; i++) table[sl[k] * W + i] = w[k][i];
                    pending[k] = false;
                } else if (prev[k] == w[k][0]) {  // duplicate build key: the generic (chained) path takes over
                    flags[FL_DUP] = 1;
                    pending[k] = false;
                } else {
                    if (++sl[k] == nslots) sl[k] = 0;
                }
                any |= pending[k];
            }
            if (++disp > MAX_DISP) { if (any) flags[FL_DISP] = 1; break; }
        }
    }
}

// ---- partitioned build: the table is cut into slot BLOCKS of 2^lgB consecutive slots, small enough for one CTA's
// shared memory.  Under linear probing a row's home slot alone decides where it can land, so a block can be built
// completely in shared memory from the rows whose home slot lies in it, and written out once with full-line stores:
// no EMPTY fill of its own, no global atomic per row, no grid barrier.
//     k_fj_build_split  packed rows (partition order) -> each block's rows, compacted at the start of the block's own
//                       slot range in `table` (a block never holds more rows than slots; the surplus is deferred)
//     k_fj_build_slab   one CTA per block: EMPTY-fill in shared memory, CAS-insert the block's rows, write the block
//     k_fj_insert       the deferred rows, into the finished table (global CAS walk from the home slot)
// A row is deferred when its probe sequence would leave its block (the slab never wraps), when its block is outside
// the window of blocks its split CTA places, or when its block is full.  Deferring is always correct: the final insert
// walks a complete table, crossing only occupied slots, so it meets an equal key (FL_DUP) before an EMPTY slot.
// Duplicate keys share a home slot; both copies end in the same block, or one of them in the deferred list.
// The direct table (DIRECT) groups the rows in a scratch area of nslots * W words instead (its table has no room for
// whole rows), and a block's rows are placed by their slots with an atomicOr on the block's bitmap words, no walk.
// Its slots are collision-free, so a block never fills up (a row beyond its block's slot count is a duplicate,
// FL_DUP) and no probe sequence leaves a block; only the window rule can defer a row, to k_fj_insert<W, true>.
constexpr int BS_THREADS = 512;
constexpr int BS_WIN = 2048;  // slot blocks one split CTA places directly
__host__ __device__ constexpr int bs_rpt(int W) { return 12 / W; }  // rows per thread and tile: 12 words in registers

template <int W>
__device__ __forceinline__ void load_row(const unsigned long long *p, unsigned long long (&w)[W]) {
    if (W == 2) {
        const int4 v = ld_stream_16(p);
        w[0] = ((unsigned long long)(unsigned)v.y << 32) | (unsigned)v.x;
        w[W - 1] = ((unsigned long long)(unsigned)v.w << 32) | (unsigned)v.z;
    } else {
#pragma unroll
        for (int i = 0; i < W; i++) w[i] = (unsigned long long)ld_stream_8(p + i);
    }
}

template <int W>
__device__ __forceinline__ void defer_row(const unsigned long long (&w)[W], unsigned long long *def, unsigned long long *ndef, int64_t def_cap,
                                          int32_t *flags) {
    const unsigned long long pos = atomicAdd(ndef, 1ULL);
    if (pos < (unsigned long long)def_cap) {
#pragma unroll
        for (int i = 0; i < W; i++) def[pos * W + i] = w[i];
    } else {
        flags[FL_DISP] = 1;  // more deferred rows than the list holds: the generic path takes over
    }
}

// One CTA per `chunk` packed rows.  Its rows lie in partitions [pa, pb] (packed order is partition order), and the home
// slot of a row of partition p lies in partition p's or p + 1's slot range (part_of reads only the hash's high 32
// bits, P <= 2^10), so the CTA's rows fall in the blocks covering slots [pa * spp, (pb + 2) * spp): its window.  Per
// tile: rank the rows per block, reserve each block's run with one global atomic on fill[block], stage the rows in
// block order in shared memory, and write every run with consecutive threads on consecutive rows.
static size_t split_smem_bytes(int W) { return (size_t)BS_THREADS * bs_rpt(W) * (W * 8 + 2); }  // stage + block of each staged row

template <int W, bool DIRECT>
__global__ void __launch_bounds__(BS_THREADS) k_fj_build_split(const unsigned long long *__restrict__ packed, int64_t rows, int64_t chunk, int P,
                                                                  uint64_t spp, uint64_t nslots, int lgB, unsigned long long *table, unsigned int *fill,
                                                                  unsigned long long *def, unsigned long long *ndef, int64_t def_cap, int32_t *flags,
                                                                  KeyMap M) {
    constexpr int R = bs_rpt(W), T = BS_THREADS * R, IPT = BS_WIN / BS_THREADS;
    extern __shared__ __align__(16) unsigned char smem_raw[];
    unsigned long long *stage = reinterpret_cast<unsigned long long *>(smem_raw);   // T * W
    unsigned short *sb = reinterpret_cast<unsigned short *>(stage + (size_t)T * W);  // T
    __shared__ unsigned int cnt[BS_WIN], start[BS_WIN], base[BS_WIN];
    __shared__ unsigned long long s_blo;
    __shared__ unsigned int s_nwin;
    typedef cub::BlockScan<unsigned int, BS_THREADS> BlockScan;
    __shared__ typename BlockScan::TempStorage scan_tmp;
    const int tid = threadIdx.x;
    const int64_t r0 = (int64_t)blockIdx.x * chunk;
    const int64_t r1 = r0 + chunk < rows ? r0 + chunk : rows;
    for (int i = tid; i < BS_WIN; i += BS_THREADS) cnt[i] = 0;
    if (tid == 0) {
        const uint64_t pa = part_of_key<DIRECT>(packed[r0 * W], P, M), pb = part_of_key<DIRECT>(packed[(r1 - 1) * W], P, M);
        uint64_t s_hi = (pb + 2) * spp;
        if (s_hi > nslots) s_hi = nslots;
        const uint64_t blo = (pa * spp) >> lgB, bhi = ((s_hi - 1) >> lgB) + 1;
        s_blo = blo;
        s_nwin = (unsigned)(bhi - blo < (uint64_t)BS_WIN ? bhi - blo : BS_WIN);
    }
    __syncthreads();
    const uint64_t blo = s_blo;
    const unsigned nwin = s_nwin;
    for (int64_t t0 = r0; t0 < r1; t0 += T) {
        const int n_tile = (int)(r1 - t0 < T ? r1 - t0 : T);
        unsigned long long w[R][W];
        unsigned int br[R], n_staged;  // window block << 16 | rank within (tile, block); T <= 2^16, BS_WIN <= 2^16
#pragma unroll
        for (int k = 0; k < R; k++)
            if (k * BS_THREADS + tid < n_tile) load_row<W>(packed + (t0 + k * BS_THREADS + tid) * W, w[k]);
#pragma unroll
        for (int k = 0; k < R; k++) {
            br[k] = 0xffffffffu;
            if (k * BS_THREADS + tid >= n_tile) continue;
            const uint64_t rel = (slot_of<DIRECT>(w[k][0], nslots, M) >> lgB) - blo;
            if (rel < nwin) {
                br[k] = ((unsigned)rel << 16) | atomicAdd(&cnt[rel], 1u);
            } else {
                defer_row<W>(w[k], def, ndef, def_cap, flags);
            }
        }
        __syncthreads();
        {  // start[] = exclusive scan of cnt[]; base[] = this tile's first position in each block's run
            unsigned int v[IPT];
#pragma unroll
            for (int i = 0; i < IPT; i++) v[i] = cnt[tid * IPT + i];
            unsigned int c[IPT];
#pragma unroll
            for (int i = 0; i < IPT; i++) c[i] = v[i];
            BlockScan(scan_tmp).ExclusiveSum(v, v, n_staged);
#pragma unroll
            for (int i = 0; i < IPT; i++) {
                const unsigned e = tid * IPT + i;
                start[e] = v[i];
                if (c[i]) {
                    base[e] = atomicAdd(&fill[blo + e], c[i]);
                    cnt[e] = 0;
                }
            }
        }
        __syncthreads();
#pragma unroll
        for (int k = 0; k < R; k++) {
            if (br[k] == 0xffffffffu) continue;
            const unsigned pos = start[br[k] >> 16] + (br[k] & 0xffffu);
#pragma unroll
            for (int i = 0; i < W; i++) stage[(size_t)pos * W + i] = w[k][i];
            sb[pos] = (unsigned short)(br[k] >> 16);
        }
        __syncthreads();
        // no barrier after the flush: stage / sb / start / base are next written after the next tile's first barrier
        for (int i = tid; i < (int)n_staged; i += BS_THREADS) {
            const unsigned e = sb[i];
            const uint64_t s0 = (blo + e) << lgB;
            const uint64_t cap = nslots - s0 < (1ull << lgB) ? nslots - s0 : (1ull << lgB);
            const uint64_t pos = (uint64_t)base[e] + (unsigned)i - start[e];
            unsigned long long rw[W];
#pragma unroll
            for (int j = 0; j < W; j++) rw[j] = stage[(size_t)i * W + j];
            if (pos >= cap) {
                if (DIRECT) flags[FL_DUP] = 1;  // more rows than distinct slots
                else defer_row<W>(rw, def, ndef, def_cap, flags);
                continue;
            }
            unsigned long long *dst = table + (s0 + pos) * W;
            if (W == 2) {
                int4 v;
                v.x = (int)(unsigned)rw[0]; v.y = (int)(unsigned)(rw[0] >> 32);
                v.z = (int)(unsigned)rw[W - 1]; v.w = (int)(unsigned)(rw[W - 1] >> 32);
                *reinterpret_cast<int4 *>(dst) = v;
            } else {
#pragma unroll
                for (int j = 0; j < W; j++) dst[j] = rw[j];
            }
        }
    }
}

// One CTA per slot block.  The block's fill[b] rows sit compacted at the start of its own slot range of `grouped`.
// Hash table (dynamic shared memory: 2^lgB * W words): `grouped` is the table itself; all of the block's rows are in
// registers before the barrier that precedes the write-out, which then overwrites that range with the finished block.
// Direct table (2^lgB * (W - 1) payload words + 2^lgB / 32 bitmap words; 2^lgB >= 32, so blocks own whole bitmap
// words): `grouped` is the split's scratch area, and the block is written to its payload range and bitmap words.
template <int W, bool DIRECT>
__global__ void __launch_bounds__(BS_THREADS) k_fj_build_slab(const unsigned long long *grouped, unsigned long long *table, uint64_t nslots, int lgB,
                                                              const unsigned int *__restrict__ fill, unsigned long long *def, unsigned long long *ndef,
                                                              int64_t def_cap, int32_t *flags, KeyMap M) {
    constexpr int R = bs_rpt(W) < 8 ? bs_rpt(W) : 8;  // the insert loop keeps its registers: no spills for W = 1
    extern __shared__ __align__(16) unsigned long long st[];
    const int tid = threadIdx.x;
    const uint64_t s0 = (uint64_t)blockIdx.x << lgB;
    const unsigned cap = (unsigned)(nslots - s0 < (1ull << lgB) ? nslots - s0 : (1ull << lgB));
    const unsigned n = fill[blockIdx.x] < cap ? fill[blockIdx.x] : cap;
    if constexpr (DIRECT) {
        constexpr int BP = W - 1;
        unsigned int *sbm = reinterpret_cast<unsigned int *>(st + (size_t)cap * BP);  // cap / 32 words
        for (unsigned i = tid; i < cap * BP; i += BS_THREADS) st[i] = 0;
        for (unsigned i = tid; i < cap / 32; i += BS_THREADS) sbm[i] = 0;
        __syncthreads();
        const unsigned long long *g = grouped + s0 * W;
        for (unsigned i0 = 0; i0 < n; i0 += BS_THREADS * R) {
            unsigned long long w[R][W];
#pragma unroll
            for (int k = 0; k < R; k++) {
                const unsigned i = i0 + k * BS_THREADS + tid;
                if (i < n) load_row<W>(g + (size_t)i * W, w[k]);
            }
#pragma unroll
            for (int k = 0; k < R; k++) {
                if (i0 + k * BS_THREADS + tid >= n) continue;
                const unsigned s = (unsigned)(slot_of<true>(w[k][0], nslots, M) - s0);  // < cap: the split grouped by block
                const unsigned int bit = 1u << (s & 31);
                if (atomicOr(sbm + (s >> 5), bit) & bit) {
                    flags[FL_DUP] = 1;
                    continue;
                }
#pragma unroll
                for (int i = 1; i < W; i++) st[(size_t)s * BP + i - 1] = w[k][i];
            }
        }
        __syncthreads();
        if (BP) {  // s0 * BP words from a 16-byte aligned base, s0 a multiple of 32: 16-byte aligned, cap * BP even
            unsigned long long *gp = table + s0 * BP;
            const int4 *s4 = reinterpret_cast<const int4 *>(st);
            for (unsigned i = tid; i < cap * BP / 2; i += BS_THREADS) st_stream_16(gp + (size_t)i * 2, s4[i]);
        }
        unsigned int *gbm = direct_bitmap<W>(table, nslots) + (s0 >> 5);
        for (unsigned i = tid; i < cap / 32; i += BS_THREADS) st_stream_4(gbm + i, (int)sbm[i]);
        return;
    }
    unsigned long long *g = table + s0 * W;
    for (unsigned i = tid; i < cap; i += BS_THREADS) {
        st[(size_t)i * W] = KEY_EMPTY;
#pragma unroll
        for (int j = 1; j < W; j++) st[(size_t)i * W + j] = 0;
    }
    __syncthreads();
    for (unsigned i0 = 0; i0 < n; i0 += BS_THREADS * R) {
        unsigned long long w[R][W];
#pragma unroll
        for (int k = 0; k < R; k++) {
            const unsigned i = i0 + k * BS_THREADS + tid;
            if (i < n) load_row<W>(g + (size_t)i * W, w[k]);
        }
#pragma unroll
        for (int k = 0; k < R; k++) {
            if (i0 + k * BS_THREADS + tid >= n) continue;
            const unsigned long long key = w[k][0];
            if (key == KEY_EMPTY) { flags[FL_SENTINEL] = 1; continue; }
            unsigned s = (unsigned)(slot_of<DIRECT>(key, nslots, M) - s0);
            int disp = 0;
            while (true) {
                if (s >= cap) { defer_row<W>(w[k], def, ndef, def_cap, flags); break; }
                const unsigned long long prev = atomicCAS(&st[(size_t)s * W], KEY_EMPTY, key);
                if (prev == KEY_EMPTY) {
#pragma unroll
                    for (int i = 1; i < W; i++) st[(size_t)s * W + i] = w[k][i];
                    break;
                }
                if (prev == key) { flags[FL_DUP] = 1; break; }
                ++s;
                if (++disp > MAX_DISP) { flags[FL_DISP] = 1; break; }
            }
        }
    }
    __syncthreads();
    const unsigned nw = cap * W;  // s0 * W words from a 16-byte aligned base, s0 even: 16-byte aligned
    const int4 *s4 = reinterpret_cast<const int4 *>(st);
    for (unsigned i = tid; i < nw / 2; i += BS_THREADS) st_stream_16(g + (size_t)i * 2, s4[i]);
    if ((nw & 1) && tid == 0) st_stream_8(g + nw - 1, (long long)st[nw - 1]);
}

// ---- probe
struct OutMap {
    void *data[GSQL_MAX_COLS * 2];
    uint8_t *nulls[GSQL_MAX_COLS * 2];
    int8_t side[GSQL_MAX_COLS * 2];  // 0 probe, 1 build
    int8_t word[GSQL_MAX_COLS * 2];
    int8_t half[GSQL_MAX_COLS * 2];
    int8_t is32[GSQL_MAX_COLS * 2];
    int32_t nout;
    int32_t join_type;
};

// ---- word-wise output staging ---------------------------------------------------------------------------------
// A tile's emitted rows are compacted into shared memory as 8-byte WORD arrays (probe words, then build payload
// words): sw[j][li].  The flush then produces each output column with 16-byte stores that are 16-byte aligned in the
// OUTPUT (groups of 4 INT32 / 2 INT64-or-FP64 elements): ~2 instructions per row-column and full-sector writes
// (unaligned warp stores reach a fraction of the HBM write rate — tools/membench.cu).
template <int R, int PW, int BP>
__device__ __forceinline__ void stage_words(char *staging, int tile_rows, bool want_flags, const unsigned long long (&pw)[R][PW],
                                            const unsigned long long (&bp)[R][BP], const bool (&found)[R], const bool (&em)[R],
                                            const unsigned int (&li)[R]) {
    unsigned long long *sw = reinterpret_cast<unsigned long long *>(staging);
    uint8_t *sf = reinterpret_cast<uint8_t *>(staging) + (size_t)(PW + BP) * tile_rows * 8;
#pragma unroll
    for (int k = 0; k < R; k++) {
        if (!em[k]) continue;
#pragma unroll
        for (int j = 0; j < PW; j++) sw[(size_t)j * tile_rows + li[k]] = pw[k][j];
#pragma unroll
        for (int j = 0; j < BP; j++) sw[(size_t)(PW + j) * tile_rows + li[k]] = found[k] ? bp[k][j] : 0ULL;
        if (want_flags) sf[li[k]] = found[k] ? 0 : 1;  // 1 = build side is NULL for this row
    }
}

// One element per lane: a warp reads 32 consecutive staged words (conflict-free) and writes one full, 128-byte
// ALIGNED line of an INT column (or two lines of a BIGINT column).  The lane -> element mapping is shifted so that
// line boundaries of the destination ADDRESS fall between warps (the column base only needs natural alignment);
// partially covered lines occur only at the two ends of the tile's run.  Everything per element is (per-column base) +
// compile-time offset: EPT unrolled stores plus one tail store for the `shift` elements the mapping pushed out.
template <int PW, int BP, int NT, int EPT>
__device__ __forceinline__ void flush_col(const OutMap &O, int q, const char *staging, unsigned long long base, int n, int32_t *flags) {
    constexpr int tile_rows = NT * EPT;
    const bool probe_side = O.side[q] == 0;
    const int j = probe_side ? O.word[q] : (O.word[q] == 0 ? 0 : PW + O.word[q] - 1);
    const char *src = staging + (size_t)j * tile_rows * 8;
    const int tid = (int)threadIdx.x;
    if (O.is32[q]) {
        int *dst = reinterpret_cast<int *>(O.data[q]) + base;
        const int l0 = tid - (int)(((unsigned long long)(uintptr_t)dst >> 2) & 31ULL);
        const unsigned int *sp = reinterpret_cast<const unsigned int *>(src) + (O.half[q] == 1 ? 1 : 0) + 2 * l0;  // element l at [2*l]
        int *dp = dst + l0;
#pragma unroll
        for (int k = 0; k < EPT; k++)
            if ((unsigned)(l0 + k * NT) < (unsigned)n) st_stream_4(dp + k * NT, (int)sp[2 * k * NT]);
        if (l0 + EPT * NT < n) st_stream_4(dp + EPT * NT, (int)sp[2 * EPT * NT]);
    } else {
        long long *dst = reinterpret_cast<long long *>(O.data[q]) + base;
        const int l0 = tid - (int)(((unsigned long long)(uintptr_t)dst >> 3) & 15ULL);
        const unsigned long long *sp = reinterpret_cast<const unsigned long long *>(src) + l0;
        long long *dp = dst + l0;
#pragma unroll
        for (int k = 0; k < EPT; k++)
            if ((unsigned)(l0 + k * NT) < (unsigned)n) st_stream_8(dp + k * NT, (long long)sp[k * NT]);
        if (l0 + EPT * NT < n) st_stream_8(dp + EPT * NT, (long long)sp[EPT * NT]);
    }
    if (O.nulls[q]) {  // NULL flags: only build-side columns of an outer join can be NULL here
        const uint8_t *sf = reinterpret_cast<const uint8_t *>(staging) + (size_t)(PW + BP) * tile_rows * 8;
        const bool outer = O.join_type == GSQL_JOIN_LEFT || O.join_type == GSQL_JOIN_RIGHT;
        uint8_t *nd = O.nulls[q] + base;
#pragma unroll
        for (int k = 0; k < EPT; k++)
            if (tid + k * NT < n) nd[tid + k * NT] = (!probe_side && outer) ? sf[tid + k * NT] : 0;
    } else if (!probe_side && (O.join_type == GSQL_JOIN_LEFT || O.join_type == GSQL_JOIN_RIGHT)) {
        if (tid == 0) flags[FL_NULLOUT] = 1;  // rejected on the host before launch
    }
}

template <int PW, int BP, int NT, int EPT>
__device__ __forceinline__ void flush_words(const OutMap &O, const char *staging, unsigned long long base, unsigned int cnt, int32_t *flags) {
    const int n = (int)cnt;
    // the first columns are unrolled: their descriptors become direct constant-bank operands
#pragma unroll
    for (int q = 0; q < 8; q++)
        if (q < O.nout) flush_col<PW, BP, NT, EPT>(O, q, staging, base, n, flags);
#pragma unroll 1
    for (int q = 8; q < O.nout; q++) flush_col<PW, BP, NT, EPT>(O, q, staging, base, n, flags);
}

static size_t stage_words_bytes(int PW, int BW, int tile_rows) {
    int BP = BW > 1 ? BW - 1 : 1;
    return (size_t)(PW + BP) * tile_rows * 8 + (size_t)tile_rows;
}

// Table lookups of the R rows a thread owns, organised in ROUNDS: every round issues the next slot read of all still
// unresolved rows before any result is consumed, so a tile costs (longest probe sequence) dependent L2 round trips
// instead of (sum over rows of the warp-wide longest sequence).  KEY_EMPTY rows (padding / the unbuildable key) never match.
// The direct table takes exactly one round and no key compare: a key in range has one possible slot, and it matches
// when that slot's bit is set (without a bitmap read when the range is dense, KeyMap).  Its payload words (L1
// bypassed) and its bitmap word (L1-cached: a partition's bitmap
// slice is at most 1/64 of its payload slice and is re-read by every row) are all requested before either is used.  The
// found flag of a row that is not live (padding, beyond the batch) is never read.
template <int R, int PW, int BW, int BP, bool DIRECT>
__device__ __forceinline__ void lookup_rounds(const unsigned long long *__restrict__ table, uint64_t nslots, uint64_t pol,
                                              const unsigned long long (&pw)[R][PW], unsigned long long (&bp)[R][BP], bool (&found)[R],
                                              const KeyMap &M) {
    uint64_t slot[R];
    unsigned long long tk[R];
    bool pending[R];
#pragma unroll
    for (int k = 0; k < R; k++) {
        slot[k] = slot_of<DIRECT>(pw[k][0], nslots, M);
#pragma unroll
        for (int i = 0; i < BP; i++) bp[k][i] = 0;
    }
    if constexpr (DIRECT) {
        const unsigned int *bm = direct_bitmap<BW>(table, nslots);
        const unsigned long long lim = M.dense ? M.dense : nslots;  // nslots = 2^bits
        unsigned int bw[R];
        bool in[R];
#pragma unroll
        for (int k = 0; k < R; k++) {
            in[k] = pw[k][0] - M.kmin < lim;
            bw[k] = 0xffffffffu;
            if (in[k]) {
                if (!M.dense) bw[k] = ld_keep_4(bm + (slot[k] >> 5), pol);
#pragma unroll
                for (int i = 0; i < BW - 1; i++) bp[k][i] = ld_keep_8_na(table + slot[k] * (BW - 1) + i, pol);
            }
        }
#pragma unroll
        for (int k = 0; k < R; k++) found[k] = in[k] && ((bw[k] >> (slot[k] & 31)) & 1u);
        return;
    }
    bool any = false;
#pragma unroll
    for (int k = 0; k < R; k++) {
        if (BW == 2) {
            int4 v = ld_keep_16_na(table + slot[k] * 2, pol);
            tk[k] = ((unsigned long long)(unsigned)v.y << 32) | (unsigned)v.x;
            bp[k][0] = ((unsigned long long)(unsigned)v.w << 32) | (unsigned)v.z;
        } else {
            tk[k] = ld_keep_8(table + slot[k] * BW, pol);
        }
    }
#pragma unroll
    for (int k = 0; k < R; k++) {
        pending[k] = pw[k][0] != KEY_EMPTY && tk[k] != pw[k][0] && tk[k] != KEY_EMPTY;
        any |= pending[k];
    }
    while (__any_sync(0xffffffffu, any)) {  // linear probing past other keys, all unresolved rows advance together
#pragma unroll
        for (int k = 0; k < R; k++) {
            if (pending[k]) {
                if (++slot[k] == nslots) slot[k] = 0;
                if (BW == 2) {
                    int4 v = ld_keep_16(table + slot[k] * 2, pol);
                    tk[k] = ((unsigned long long)(unsigned)v.y << 32) | (unsigned)v.x;
                    bp[k][0] = ((unsigned long long)(unsigned)v.w << 32) | (unsigned)v.z;
                } else {
                    tk[k] = ld_keep_8(table + slot[k] * BW, pol);
                }
            }
        }
        any = false;
#pragma unroll
        for (int k = 0; k < R; k++) {
            pending[k] = pending[k] && tk[k] != pw[k][0] && tk[k] != KEY_EMPTY;
            any |= pending[k];
        }
    }
#pragma unroll
    for (int k = 0; k < R; k++) {
        found[k] = pw[k][0] != KEY_EMPTY && tk[k] == pw[k][0];
        if (BW > 2 && found[k]) {
#pragma unroll
            for (int i = 1; i < BW; i++) bp[k][i - 1] = ld_keep_8(table + slot[k] * BW + i, pol);
        }
    }
}

struct ProbeShared {
    unsigned int cell[THREADS / 32][RPT];
    unsigned long long tile_base;
    unsigned int tile_total;
};

// Steps 2-4 of a probe tile, given the RPT packed probe rows of this thread in pw (rows beyond the batch carry KEY_EMPTY
// and live[k] = false): table lookups, emit decision, tile-wide compaction, staged column flush.
template <int PW, int BW, bool DIRECT>
__device__ __forceinline__ void probe_tile(unsigned long long (&pw)[RPT][PW], const bool (&live)[RPT], const unsigned long long *__restrict__ table,
                                           uint64_t nslots, uint64_t pol, const OutMap &O, unsigned long long *cursor, int32_t *flags,
                                           ProbeShared &sh, unsigned char *probe_stage, const KeyMap &M) {
    constexpr int BP = BW > 1 ? BW - 1 : 1;
    const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
    unsigned long long bp[RPT][BP];  // build payload words (the build key equals the probe key on a match)
    unsigned int ballot[RPT];
    bool found[RPT];
    // 2. table lookups in rounds (one L2-resident read per row per round, all rows of the thread in flight)
    lookup_rounds<RPT, PW, BW, BP, DIRECT>(table, nslots, pol, pw, bp, found, M);
    // 3. which rows emit (AbstractBufferedJoinExec.nextRows:185-264 for unique build keys, no NULLs)
#pragma unroll
    for (int k = 0; k < RPT; k++) {
        bool emit;
        switch (O.join_type) {
        case GSQL_JOIN_INNER: emit = found[k]; break;
        case GSQL_JOIN_SEMI: emit = found[k]; break;
        case GSQL_JOIN_ANTI: emit = !found[k]; break;
        default: emit = true; break;  // LEFT / RIGHT: unmatched probe rows are NULL-padded
        }
        emit = emit && live[k];
        ballot[k] = __ballot_sync(0xffffffffu, emit);
        if (lane == 0) sh.cell[warp][k] = __popc(ballot[k]);
    }
    __syncthreads();
    unsigned long long my_base = 0;
    if (warp == 0) {  // exclusive scan over the 64 (warp, k) cells + one cursor bump for the tile
        constexpr int CELLS = (THREADS / 32) * RPT;
        unsigned int *flat = &sh.cell[0][0];
        unsigned int a = flat[lane * 2], b = flat[lane * 2 + 1];
        unsigned int sum = a + b, incl = sum;
#pragma unroll
        for (int d = 1; d < 32; d <<= 1) {
            unsigned int t = __shfl_up_sync(0xffffffffu, incl, d);
            if (lane >= d) incl += t;
        }
        unsigned int excl = incl - sum;
        unsigned int total = __shfl_sync(0xffffffffu, incl, 31);
        if (lane == 0) {  // the cursor bump's round trip overlaps the staging below: its result is only published after it
            my_base = total ? atomicAdd(cursor, (unsigned long long)total) : 0ULL;
            sh.tile_total = total;
        }
        flat[lane * 2] = excl;
        flat[lane * 2 + 1] = excl + a;
        static_assert(CELLS == 64, "cell scan assumes 64 cells");
    }
    __syncthreads();
    // 4. compact the tile's rows into shared memory (word arrays), then flush the columns with aligned full-line stores
    const bool want_flags = O.join_type == GSQL_JOIN_LEFT || O.join_type == GSQL_JOIN_RIGHT;
    bool em[RPT];
    unsigned int li[RPT];
#pragma unroll
    for (int k = 0; k < RPT; k++) {
        em[k] = (ballot[k] >> lane) & 1u;
        li[k] = sh.cell[warp][k] + __popc(ballot[k] & ((1u << lane) - 1u));
    }
    stage_words<RPT, PW, BP>(reinterpret_cast<char *>(probe_stage), TILE, want_flags, pw, bp, found, em, li);
    if (threadIdx.x == 0) sh.tile_base = my_base;
    __syncthreads();
    flush_words<PW, BP, THREADS, RPT>(O, reinterpret_cast<const char *>(probe_stage), sh.tile_base, sh.tile_total, flags);
}

// One tile per block; probe rows come from the input columns (packed == nullptr) or from packed rows.  gaps: the packed
// rows are the one-pass region layout, whose KEY_EMPTY rows are padding (never emitted); when its partition spilled,
// the layout is incomplete and the kernel does nothing.
template <int PW, int BW, bool DIRECT>
__global__ void __launch_bounds__(THREADS, 2) k_fj_probe(const unsigned long long *__restrict__ packed, const __grid_constant__ DColSet cols,
                                                      const __grid_constant__ Layout L, int64_t n, bool gaps, const unsigned long long *__restrict__ table,
                                                      uint64_t nslots, const __grid_constant__ OutMap O, unsigned long long *cursor, int32_t *flags,
                                                      KeyMap M) {
    __shared__ ProbeShared sh;
    extern __shared__ __align__(16) unsigned char probe_stage[];
    if (gaps && *(volatile int32_t *)(flags + FL_SPILL)) return;
    const uint64_t pol = l2_policy_evict_last();
    const int64_t t0 = (int64_t)blockIdx.x * TILE;
    unsigned long long pw[RPT][PW];
    bool live[RPT];
    // 1. stream the probe rows in (all RPT loads in flight)
    if (packed) {
#pragma unroll
        for (int k = 0; k < RPT; k++) {
            int64_t r = t0 + k * THREADS + threadIdx.x;
            if (r < n) {
                if (PW == 2) {
                    int4 v = ld_stream_16(packed + r * 2);
                    pw[k][0] = ((unsigned long long)(unsigned)v.y << 32) | (unsigned)v.x;
                    pw[k][PW - 1] = ((unsigned long long)(unsigned)v.w << 32) | (unsigned)v.z;
                } else {
#pragma unroll
                    for (int i = 0; i < PW; i++) pw[k][i] = (unsigned long long)ld_stream_8(packed + r * PW + i);
                }
            } else {
#pragma unroll
                for (int i = 0; i < PW; i++) pw[k][i] = 0;
            }
        }
    } else {
        pack_tile<PW>(cols, L, t0 + threadIdx.x, n, pw);
    }
#pragma unroll
    for (int k = 0; k < RPT; k++) {
        live[k] = t0 + k * THREADS + threadIdx.x < n && !(gaps && pw[k][0] == KEY_EMPTY);
        if (!live[k]) pw[k][0] = KEY_EMPTY;
    }
    probe_tile<PW, BW, DIRECT>(pw, live, table, nslots, pol, O, cursor, flags, sh, probe_stage, M);
}

}  // namespace fj

struct JoinFast {
    bool eligible = false;   // decided at create: shape supports the packed single-key path
    bool enabled = false;    // table built and usable
    fj::Layout bl, pl;       // build / probe packed-row layouts
    int P = 1;               // partitions (1 = table small enough to stay in L2 without partitioning)
    uint64_t nslots = 0;
    bool direct = false;     // the direct table (dense build keys, fj::KeyMap) instead of the hash table
    fj::KeyMap km{};
    DevBuf table, flags, cursor;
    // tuning switches read by fast_build (INTEGRATION §7); these are their defaults
    int64_t part_bytes = 16ll << 20;
    int64_t sub_batch = 1ll << 30;  // probe rows per partition+probe round (bounds scratch memory)
    int64_t part_min_rows = 1ll << 20;  // smaller probe batches skip the partitioning passes
};
