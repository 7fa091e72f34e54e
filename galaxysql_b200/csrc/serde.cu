// serde.cu — the MPP wire codec of a Chunk on the GPU (SURVEY §8f rank 3), behind gsql_serde_*.
//
// Reference path restated (EX/ = polardbx-executor/src/main/java/com/alibaba/polardbx/executor/):
//   EX/mpp/execution/buffer/PagesSerde.java:57-115 (serialize / deserialize, uncompressed path)
//   EX/mpp/execution/buffer/PagesSerdeUtil.java:36-67 (writeRawPage / readRawPage / SerializedChunk framing)
//   EX/chunk/IntegerBlockEncoding.java:46-70, LongBlockEncoding.java:47-73, DoubleBlockEncoding.java:46-70
//   EX/chunk/EncoderUtil.java:43-150 (NULL flags as a bit stream, first row in the most significant bit)
// The reference walks a chunk row by row through SliceOutput; here one thread block encodes (decodes) one page:
// a first kernel counts the non-NULL values per (page, column), an exclusive scan turns the page sizes into byte
// offsets, and the page kernel writes header, bit stream and the compacted values (block-wide prefix sum of the
// non-NULL flags).  The byte stream is unaligned by construction (13-byte frame headers, bit streams of any length), so
// values are stored byte-wise; this path is bound by the host link it feeds, not by HBM.
#include <cub/block/block_scan.cuh>
#include <cub/device/device_reduce.cuh>
#include <cub/device/device_scan.cuh>

#include <stdint.h>
#include <vector>

#include "common.cuh"

namespace {

constexpr int SD_THREADS = 256;
constexpr int FRAME_BYTES = 13;  // positionCount, marker, uncompressedSize, sizeInBytes

struct SerdeCols {
    DColSet in;
    int64_t rows;
    int32_t page_rows, npages;
};

__device__ __forceinline__ int64_t page_payload_bytes(const SerdeCols &S, const int64_t *nonnull, int64_t page, int m) {
    int64_t b = 4;  // blockCount
    for (int c = 0; c < S.in.n; c++) b += 4 + (m + 7) / 8 + nonnull[page * S.in.n + c] * gsql_type_width(S.in.c[c].type);
    return b;
}

// nonnull[page * ncols + c] = non-NULL rows of column c in the page; size[page] = framed page bytes
__global__ void __launch_bounds__(SD_THREADS) k_serde_count(const __grid_constant__ SerdeCols S, int64_t *__restrict__ nonnull, int64_t *__restrict__ size) {
    __shared__ int cnt[GSQL_MAX_COLS];
    for (int64_t page = blockIdx.x; page < S.npages; page += gridDim.x) {
        const int64_t r0 = page * S.page_rows;
        const int m = (int)(S.rows - r0 < S.page_rows ? S.rows - r0 : S.page_rows);
        if (threadIdx.x < S.in.n) cnt[threadIdx.x] = 0;
        __syncthreads();
        for (int c = 0; c < S.in.n; c++) {
            const uint8_t *nl = S.in.c[c].nulls;
            int mine = 0;
            if (nl)
                for (int i = threadIdx.x; i < m; i += SD_THREADS) mine += nl[r0 + i] ? 1 : 0;
            if (mine) atomicAdd(&cnt[c], mine);
        }
        __syncthreads();
        if (threadIdx.x < S.in.n) nonnull[page * S.in.n + threadIdx.x] = m - cnt[threadIdx.x];
        __syncthreads();
        if (threadIdx.x == 0) size[page] = FRAME_BYTES + page_payload_bytes(S, nonnull, page, m);
        __syncthreads();
    }
}

__device__ __forceinline__ void put_le(uint8_t *p, unsigned long long v, int w) {
    for (int i = 0; i < w; i++) p[i] = (uint8_t)(v >> (8 * i));
}
__device__ __forceinline__ unsigned long long get_le(const uint8_t *p, int w) {
    unsigned long long v = 0;
    for (int i = 0; i < w; i++) v |= (unsigned long long)p[i] << (8 * i);
    return v;
}

__global__ void __launch_bounds__(SD_THREADS) k_serde_encode(const __grid_constant__ SerdeCols S, const int64_t *__restrict__ nonnull,
                                                             const int64_t *__restrict__ offs, uint8_t *__restrict__ out) {
    typedef cub::BlockScan<int, SD_THREADS> BlockScan;
    __shared__ typename BlockScan::TempStorage scan_tmp;
    __shared__ int carry;
    for (int64_t page = blockIdx.x; page < S.npages; page += gridDim.x) {
        const int64_t r0 = page * S.page_rows;
        const int m = (int)(S.rows - r0 < S.page_rows ? S.rows - r0 : S.page_rows);
        uint8_t *p = out + offs[page];
        const int64_t payload = page_payload_bytes(S, nonnull, page, m);
        if (threadIdx.x == 0) {  // SerializedChunk frame (PagesSerdeUtil.writeSerializedChunk:50-58) + blockCount
            put_le(p, (unsigned)m, 4);
            p[4] = 0;  // ChunkCompression.UNCOMPRESSED
            put_le(p + 5, (unsigned long long)payload, 4);
            put_le(p + 9, (unsigned long long)payload, 4);
            put_le(p + FRAME_BYTES, (unsigned)S.in.n, 4);
        }
        uint8_t *q = p + FRAME_BYTES + 4;
        for (int c = 0; c < S.in.n; c++) {
            const DCol &col = S.in.c[c];
            const int w = gsql_type_width(col.type);
            if (threadIdx.x == 0) put_le(q, (unsigned)m, 4);
            uint8_t *bits = q + 4;
            uint8_t *vals = bits + (m + 7) / 8;
            // NULL flags as a bit stream: one thread per output byte (EncoderUtil.encodeNullsAsBits:43-110)
            for (int b = threadIdx.x; b < (m + 7) / 8; b += SD_THREADS) {
                unsigned v = 0;
                for (int k = 0; k < 8; k++) {
                    const int i = b * 8 + k;
                    if (i < m && col.nulls && col.nulls[r0 + i]) v |= 0x80u >> k;
                }
                bits[b] = (uint8_t)v;
            }
            // non-NULL values, compacted in row order
            if (threadIdx.x == 0) carry = 0;
            __syncthreads();
            for (int base = 0; base < m; base += SD_THREADS) {
                const int i = base + threadIdx.x;
                const bool live = i < m && !(col.nulls && col.nulls[r0 + i]);
                int pos;
                int total;
                BlockScan(scan_tmp).ExclusiveSum(live ? 1 : 0, pos, total);
                const int start = carry;
                if (live) {
                    unsigned long long v = w == 4 ? (unsigned long long)(unsigned)reinterpret_cast<const int *>(col.data)[r0 + i]
                                                  : (unsigned long long)reinterpret_cast<const long long *>(col.data)[r0 + i];
                    put_le(vals + (size_t)(start + pos) * w, v, w);
                }
                __syncthreads();
                if (threadIdx.x == 0) carry = start + total;
                __syncthreads();
            }
            q = vals + (size_t)nonnull[page * S.in.n + c] * w;
        }
        __syncthreads();
    }
}

struct DecodeOut {
    void *data[GSQL_MAX_COLS];
    uint8_t *nulls[GSQL_MAX_COLS];
    int32_t types[GSQL_MAX_COLS];
    int32_t ncols;
};

// One block per page.  page_off[page] = byte offset of the page's frame, row_off[page] = first output row.  The host has
// checked every block of every page against its page's sizeInBytes (serde_check_page), so no read leaves the page.
__global__ void __launch_bounds__(SD_THREADS) k_serde_decode(const uint8_t *__restrict__ bytes, const int64_t *__restrict__ page_off,
                                                             const int64_t *__restrict__ row_off, int64_t npages, const __grid_constant__ DecodeOut O) {
    typedef cub::BlockScan<int, SD_THREADS> BlockScan;
    __shared__ typename BlockScan::TempStorage scan_tmp;
    __shared__ int carry;
    for (int64_t page = blockIdx.x; page < npages; page += gridDim.x) {
        const uint8_t *p = bytes + page_off[page];
        const int m = (int)get_le(p, 4);
        const int64_t r0 = row_off[page];
        const uint8_t *q = p + FRAME_BYTES + 4;
        for (int c = 0; c < O.ncols; c++) {
            const int w = gsql_type_width(O.types[c]);
            const uint8_t *bits = q + 4;
            const uint8_t *vals = bits + (m + 7) / 8;
            if (threadIdx.x == 0) carry = 0;
            __syncthreads();
            for (int base = 0; base < m; base += SD_THREADS) {
                const int i = base + threadIdx.x;
                const bool isnull = i < m && ((bits[i >> 3] >> (7 - (i & 7))) & 1);  // EncoderUtil.decodeNullBits:116-150
                const bool live = i < m && !isnull;
                int pos, total;
                BlockScan(scan_tmp).ExclusiveSum(live ? 1 : 0, pos, total);
                const int start = carry;
                if (i < m) {
                    O.nulls[c][r0 + i] = isnull ? 1 : 0;
                    const unsigned long long v = live ? get_le(vals + (size_t)(start + pos) * w, w) : 0ULL;
                    if (w == 4) reinterpret_cast<int *>(O.data[c])[r0 + i] = (int)(unsigned)v;
                    else reinterpret_cast<long long *>(O.data[c])[r0 + i] = (long long)v;
                }
                __syncthreads();
                if (threadIdx.x == 0) carry = start + total;
                __syncthreads();
            }
            q = vals + (size_t)carry * w;
            __syncthreads();
        }
    }
}

struct SerdePlan {
    SerdeCols S;
    StagedBatch sb;
    DevBuf nonnull, size, offs, tmp;
    int64_t total = 0;
};

gsql_status serde_plan(gsql_ctx *ctx, const gsql_batch *in, int32_t page_rows, SerdePlan *P) {
    GSQL_TRY(validate_batch(ctx, in, -1, nullptr));
    if (page_rows < 1) return gsql_set_error(ctx, GSQL_E_INVALID, "page_rows must be positive");
    for (int i = 0; i < in->ncols; i++)
        if (in->cols[i].type == GSQL_T_DEC128) return gsql_set_error(ctx, GSQL_E_UNSUPPORTED, "DEC128 columns have no block encoding here");
    GSQL_CUDA(ctx, cudaSetDevice(ctx->device));
    GSQL_TRY(stage_batch(ctx, in, &P->sb));
    memset(&P->S, 0, sizeof(P->S));
    P->S.in.n = in->ncols;
    for (int i = 0; i < in->ncols; i++) P->S.in.c[i] = P->sb.cols[i];
    P->S.rows = in->rows;
    P->S.page_rows = page_rows;
    const int64_t npages = div_up(in->rows, page_rows);
    if (npages > 0x7fffffff) return gsql_set_error(ctx, GSQL_E_UNSUPPORTED, "too many pages");
    P->S.npages = (int32_t)npages;
    P->total = 0;
    if (npages == 0) return GSQL_OK;
    GSQL_TRY(P->nonnull.alloc(ctx, (size_t)npages * in->ncols * 8 + 8));
    GSQL_TRY(P->size.alloc(ctx, (size_t)(npages + 1) * 8));
    GSQL_TRY(P->offs.alloc(ctx, (size_t)(npages + 1) * 8));
    GSQL_CUDA(ctx, cudaMemsetAsync((char *)P->size.p + npages * 8, 0, 8, ctx->stream));
    {
        KernelScope ks(ctx, "serde_count");
        int grid = (int)(npages < (int64_t)ctx->sm_count * 8 ? npages : (int64_t)ctx->sm_count * 8);
        k_serde_count<<<grid, SD_THREADS, 0, ctx->stream>>>(P->S, P->nonnull.as<int64_t>(), P->size.as<int64_t>());
    }
    GSQL_CUDA(ctx, cudaGetLastError());
    size_t tb = 0;
    GSQL_CUDA(ctx, cub::DeviceScan::ExclusiveSum(nullptr, tb, P->size.as<int64_t>(), P->offs.as<int64_t>(), npages + 1, ctx->stream));
    GSQL_TRY(P->tmp.alloc(ctx, tb));
    GSQL_CUDA(ctx, cub::DeviceScan::ExclusiveSum(P->tmp.p, tb, P->size.as<int64_t>(), P->offs.as<int64_t>(), npages + 1, ctx->stream));
    GSQL_CUDA(ctx, cudaMemcpyAsync(&P->total, P->offs.as<int64_t>() + npages, 8, cudaMemcpyDeviceToHost, ctx->stream));
    // uncompressedSize and sizeInBytes are int32 fields: a page whose payload could pass INT32_MAX (counted without NULLs)
    // has its exact framed size checked
    int64_t bound = 4;
    for (int i = 0; i < in->ncols; i++) bound += 4 + ((int64_t)page_rows + 7) / 8 + (int64_t)page_rows * gsql_type_width(in->cols[i].type);
    int64_t biggest = 0;
    if (bound > INT32_MAX) {
        DevBuf dmax, mtmp;
        GSQL_TRY(dmax.alloc(ctx, 8));
        size_t mb = 0;
        GSQL_CUDA(ctx, cub::DeviceReduce::Max(nullptr, mb, P->size.as<int64_t>(), dmax.as<int64_t>(), npages, ctx->stream));
        GSQL_TRY(mtmp.alloc(ctx, mb));
        GSQL_CUDA(ctx, cub::DeviceReduce::Max(mtmp.p, mb, P->size.as<int64_t>(), dmax.as<int64_t>(), npages, ctx->stream));
        GSQL_CUDA(ctx, cudaMemcpyAsync(&biggest, dmax.p, 8, cudaMemcpyDeviceToHost, ctx->stream));
    }
    GSQL_CUDA(ctx, cudaStreamSynchronize(ctx->stream));
    if (biggest - FRAME_BYTES > INT32_MAX)
        return gsql_set_error(ctx, GSQL_E_UNSUPPORTED, "a page of %d rows needs %lld payload bytes; the frame's sizeInBytes is an int32", page_rows,
                              (long long)(biggest - FRAME_BYTES));
    return GSQL_OK;
}

// Checks one page against the reference's reader, which decodes a page from a slice bounded by its sizeInBytes
// (PagesSerdeUtil.readRawPage): the block count, then per block the positionCount, the NULL bit stream and as many values
// as it has clear bits must all lie inside the page.  Bytes left after the last block are ignored, as the reference
// ignores them.  p = the page's first payload byte (blockCount), sz = sizeInBytes, m = the frame's positionCount.
bool serde_check_page(const uint8_t *p, int64_t sz, int64_t m, const DecodeOut &O, const char **why) {
    auto rd32 = [&](int64_t o) -> int64_t { return (int64_t)(int32_t)((uint32_t)p[o] | (uint32_t)p[o + 1] << 8 | (uint32_t)p[o + 2] << 16 | (uint32_t)p[o + 3] << 24); };
    if (rd32(0) != O.ncols) return *why = "block count differs from the schema", false;
    const int64_t nbits = (m + 7) / 8;
    int64_t q = 4;
    for (int c = 0; c < O.ncols; c++) {
        if (q + 4 > sz) return *why = "block header past the page end", false;
        if (rd32(q) != m) return *why = "block positionCount differs from the page's", false;
        q += 4;
        if (q + nbits > sz) return *why = "NULL bit stream past the page end", false;
        int64_t nulls = 0;
        for (int64_t b = 0; b < nbits; b++) {
            unsigned v = p[q + b];
            if (b == nbits - 1 && (m & 7)) v &= 0xffu << (8 - (m & 7));  // the padding bits of the last byte are not rows
            nulls += __builtin_popcount(v);
        }
        q += nbits;
        const int64_t vbytes = (m - nulls) * gsql_type_width(O.types[c]);
        if (q + vbytes > sz) return *why = "values past the page end", false;
        q += vbytes;
    }
    return true;
}

}  // namespace

extern "C" gsql_status gsql_serde_size(gsql_ctx *ctx, const gsql_batch *in, int32_t page_rows, int64_t *bytes) {
    if (!ctx || !in || !bytes) return GSQL_E_INVALID;
    if (ctx->sticky) return GSQL_E_CUDA;
    SerdePlan P;
    GSQL_TRY(serde_plan(ctx, in, page_rows, &P));
    *bytes = P.total;
    return GSQL_OK;
}

extern "C" gsql_status gsql_serde_serialize(gsql_ctx *ctx, const gsql_batch *in, int32_t page_rows, void *out_bytes, int64_t capacity, int64_t *bytes) {
    if (!ctx || !in || !bytes) return GSQL_E_INVALID;
    if (ctx->sticky) return GSQL_E_CUDA;
    SerdePlan P;
    GSQL_TRY(serde_plan(ctx, in, page_rows, &P));
    *bytes = P.total;
    if (P.total > capacity) return gsql_set_error(ctx, GSQL_E_CAPACITY, "serialized batch needs %lld bytes, capacity %lld", (long long)P.total, (long long)capacity);
    if (P.total == 0) return GSQL_OK;
    if (!out_bytes) return gsql_set_error(ctx, GSQL_E_INVALID, "null output buffer");
    DevBuf dout;
    uint8_t *d_out = (uint8_t *)out_bytes;
    if (in->mem == GSQL_MEM_HOST) {
        GSQL_TRY(dout.alloc(ctx, (size_t)P.total));
        d_out = dout.as<uint8_t>();
    }
    {
        KernelScope ks(ctx, "serde_encode");
        int64_t npages = P.S.npages;
        int grid = (int)(npages < (int64_t)ctx->sm_count * 8 ? npages : (int64_t)ctx->sm_count * 8);
        k_serde_encode<<<grid, SD_THREADS, 0, ctx->stream>>>(P.S, P.nonnull.as<int64_t>(), P.offs.as<int64_t>(), d_out);
    }
    GSQL_CUDA(ctx, cudaGetLastError());
    if (in->mem == GSQL_MEM_HOST) GSQL_CUDA(ctx, cudaMemcpyAsync(out_bytes, d_out, (size_t)P.total, cudaMemcpyDeviceToHost, ctx->stream));
    GSQL_CUDA(ctx, cudaStreamSynchronize(ctx->stream));
    return GSQL_OK;
}

extern "C" gsql_status gsql_serde_deserialize(gsql_ctx *ctx, const void *bytes, int64_t nbytes, int32_t mem, gsql_batch *out, int64_t out_capacity,
                                              int64_t *out_rows) {
    if (!ctx || !out || !out_rows || nbytes < 0 || (nbytes > 0 && !bytes)) return GSQL_E_INVALID;
    if (ctx->sticky) return GSQL_E_CUDA;
    GSQL_TRY(validate_batch(ctx, out, -1, nullptr));
    if (out->mem != mem) return gsql_set_error(ctx, GSQL_E_INVALID, "bytes and out must live in the same memory space");
    for (int c = 0; c < out->ncols; c++) {
        if (out->cols[c].type == GSQL_T_DEC128) return gsql_set_error(ctx, GSQL_E_UNSUPPORTED, "DEC128 columns have no block encoding here");
        if (out_capacity > 0 && !out->cols[c].nulls) return gsql_set_error(ctx, GSQL_E_INVALID, "output column %d needs a nulls buffer", c);
    }
    GSQL_CUDA(ctx, cudaSetDevice(ctx->device));
    *out_rows = 0;
    out->rows = 0;
    if (nbytes == 0) return GSQL_OK;
    DecodeOut O;
    memset(&O, 0, sizeof(O));
    O.ncols = out->ncols;
    for (int c = 0; c < out->ncols; c++) O.types[c] = out->cols[c].type;
    // ---- every page and every block is checked on the host before the capacity verdict and before any launch (sizeInBytes
    //      chains the pages; a device batch downloads its bytes first)
    std::vector<uint8_t> hostcopy;
    const uint8_t *hb = (const uint8_t *)bytes;
    if (mem == GSQL_MEM_DEVICE) {
        hostcopy.resize((size_t)nbytes);
        GSQL_CUDA(ctx, cudaMemcpyAsync(hostcopy.data(), bytes, (size_t)nbytes, cudaMemcpyDeviceToHost, ctx->stream));
        GSQL_CUDA(ctx, cudaStreamSynchronize(ctx->stream));
        hb = hostcopy.data();
    }
    auto rd32 = [&](int64_t o) -> int64_t { return (int64_t)(int32_t)((uint32_t)hb[o] | (uint32_t)hb[o + 1] << 8 | (uint32_t)hb[o + 2] << 16 | (uint32_t)hb[o + 3] << 24); };
    std::vector<int64_t> page_off, row_off;
    int64_t pos = 0, rows = 0;
    while (pos < nbytes) {
        if (pos + FRAME_BYTES > nbytes) return gsql_set_error(ctx, GSQL_E_INVALID, "truncated page frame at byte %lld", (long long)pos);
        const int64_t m = rd32(pos), unc = rd32(pos + 5), sz = rd32(pos + 9);
        const int marker = hb[pos + 4];
        if (marker != 0) return gsql_set_error(ctx, GSQL_E_INVALID, "compressed page at byte %lld (ChunkCompression marker %d)", (long long)pos, marker);
        if (m < 0 || sz < 4 || unc != sz || pos + FRAME_BYTES + sz > nbytes) return gsql_set_error(ctx, GSQL_E_INVALID, "corrupt page frame at byte %lld", (long long)pos);
        const char *why = "";
        if (!serde_check_page(hb + pos + FRAME_BYTES, sz, m, O, &why))
            return gsql_set_error(ctx, GSQL_E_INVALID, "page at byte %lld does not match the schema: %s", (long long)pos, why);
        page_off.push_back(pos);
        row_off.push_back(rows);
        rows += m;
        pos += FRAME_BYTES + sz;
    }
    *out_rows = rows;
    if (rows > out_capacity) return gsql_set_error(ctx, GSQL_E_CAPACITY, "pages hold %lld rows, capacity %lld", (long long)rows, (long long)out_capacity);
    const int64_t npages = (int64_t)page_off.size();
    DevBuf dbytes, dpoff, droff;
    const uint8_t *d_bytes = (const uint8_t *)bytes;
    if (mem == GSQL_MEM_HOST) {
        GSQL_TRY(dbytes.alloc(ctx, (size_t)nbytes));
        GSQL_CUDA(ctx, cudaMemcpyAsync(dbytes.p, bytes, (size_t)nbytes, cudaMemcpyHostToDevice, ctx->stream));
        d_bytes = dbytes.as<uint8_t>();
    }
    GSQL_TRY(dpoff.alloc(ctx, (size_t)npages * 8));
    GSQL_TRY(droff.alloc(ctx, (size_t)npages * 8));
    GSQL_CUDA(ctx, cudaMemcpyAsync(dpoff.p, page_off.data(), (size_t)npages * 8, cudaMemcpyHostToDevice, ctx->stream));
    GSQL_CUDA(ctx, cudaMemcpyAsync(droff.p, row_off.data(), (size_t)npages * 8, cudaMemcpyHostToDevice, ctx->stream));
    OutBinding ob;
    GSQL_TRY(out_bind(ctx, out, rows, &ob));
    for (int c = 0; c < out->ncols; c++) {
        O.data[c] = ob.data[c];
        O.nulls[c] = ob.nulls[c];
    }
    {
        KernelScope ks(ctx, "serde_decode");
        int grid = (int)(npages < (int64_t)ctx->sm_count * 8 ? npages : (int64_t)ctx->sm_count * 8);
        k_serde_decode<<<grid, SD_THREADS, 0, ctx->stream>>>(d_bytes, dpoff.as<int64_t>(), droff.as<int64_t>(), npages, O);
    }
    GSQL_CUDA(ctx, cudaGetLastError());
    GSQL_TRY(out_download(ctx, out, rows, ob));  // synchronises a host batch with rows; every other call synchronises here
    if (mem == GSQL_MEM_DEVICE || rows == 0) GSQL_CUDA(ctx, cudaStreamSynchronize(ctx->stream));
    out->rows = rows;
    return GSQL_OK;
}
