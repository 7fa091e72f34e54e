// ctx.cu — context, error plumbing, stream-ordered memory, batch staging, the row store and output binding, per-kernel event timing,
// and the two contractual hash utilities (gsql_hash_rows / gsql_partition_ids).
#include <stdarg.h>

#include "common.cuh"

gsql_status gsql_set_error(gsql_ctx *ctx, gsql_status st, const char *fmt, ...) {
    if (ctx) {
        va_list ap;
        va_start(ap, fmt);
        vsnprintf(ctx->err, sizeof(ctx->err), fmt, ap);
        va_end(ap);
    }
    return st;
}

extern "C" int gsql_abi_version(void) { return GSQL_ABI_VERSION; }

extern "C" gsql_status gsql_ctx_create(int device, gsql_ctx **out) {
    if (!out) return GSQL_E_INVALID;
    *out = nullptr;
    int count = 0;
    cudaError_t e = cudaGetDeviceCount(&count);
    if (e != cudaSuccess || count == 0 || device < 0 || device >= count) {
        // No CPU fallback exists behind this ABI: fail loudly.
        fprintf(stderr, "libgsql_gpu: no usable CUDA device %d (%s)\n", device,
                e != cudaSuccess ? cudaGetErrorString(e) : "device index out of range");
        return GSQL_E_CUDA;
    }
    gsql_ctx *ctx = new gsql_ctx();
    ctx->device = device;
    if (cudaSetDevice(device) != cudaSuccess) { delete ctx; return GSQL_E_CUDA; }
    if (cudaStreamCreateWithFlags(&ctx->stream, cudaStreamNonBlocking) != cudaSuccess) { delete ctx; return GSQL_E_CUDA; }
    ctx->own_stream = true;
    cudaStreamCreateWithFlags(&ctx->copy_in, cudaStreamNonBlocking);
    cudaStreamCreateWithFlags(&ctx->copy_out, cudaStreamNonBlocking);
    cudaDeviceGetAttribute(&ctx->sm_count, cudaDevAttrMultiProcessorCount, device);
    // Random 16-byte hash-table reads: with the default L2 fetch granularity every miss pulled a whole 128-byte line
    // from HBM, about three times the useful sectors.  Ask for 32-byte sector fetches.
    {
        int gran = 32;
        env_knob("GSQL_L2_FETCH_GRANULARITY", &gran);
        if (gran == 32 || gran == 64 || gran == 128) cudaDeviceSetLimit(cudaLimitMaxL2FetchGranularity, (size_t)gran);
        cudaGetLastError();
    }
    // keep freed blocks in the pool: operators allocate/free tables repeatedly
    cudaMemPool_t pool;
    if (cudaDeviceGetDefaultMemPool(&pool, device) == cudaSuccess) {
        uint64_t thr = UINT64_MAX;
        cudaMemPoolSetAttribute(pool, cudaMemPoolAttrReleaseThreshold, &thr);
    }
    *out = ctx;
    return GSQL_OK;
}

#include <mutex>
static std::mutex g_ref_mutex;

void gsql_ctx_retain(gsql_ctx *ctx) {
    std::lock_guard<std::mutex> g(g_ref_mutex);
    ctx->refs++;
}

static void ctx_teardown(gsql_ctx *ctx);

void gsql_ctx_release(gsql_ctx *ctx) {
    bool last;
    {
        std::lock_guard<std::mutex> g(g_ref_mutex);
        last = --ctx->refs == 0;
    }
    if (last) ctx_teardown(ctx);
}

// The context's resources live until the last handle created on it is destroyed.
extern "C" void gsql_ctx_destroy(gsql_ctx *ctx) {
    if (!ctx) return;
    gsql_ctx_release(ctx);
}

static void ctx_teardown(gsql_ctx *ctx) {
    cudaSetDevice(ctx->device);
    cudaStreamSynchronize(ctx->stream);
    for (auto &p : ctx->prof)
        for (auto &ev : p.pending) { cudaEventDestroy(ev.first); cudaEventDestroy(ev.second); }
    for (auto ev : ctx->event_pool) cudaEventDestroy(ev);
    if (ctx->own_stream) cudaStreamDestroy(ctx->stream);
    if (ctx->copy_in) cudaStreamDestroy(ctx->copy_in);
    if (ctx->copy_out) cudaStreamDestroy(ctx->copy_out);
    delete ctx;
}

extern "C" const char *gsql_last_error(const gsql_ctx *ctx) { return ctx ? ctx->err : "null context"; }

extern "C" gsql_status gsql_ctx_sync(gsql_ctx *ctx) {
    if (!ctx) return GSQL_E_INVALID;
    GSQL_CUDA(ctx, cudaStreamSynchronize(ctx->stream));
    return GSQL_OK;
}

extern "C" void *gsql_ctx_stream(gsql_ctx *ctx) { return ctx ? (void *)ctx->stream : nullptr; }

extern "C" gsql_status gsql_ctx_set_stream(gsql_ctx *ctx, void *s) {
    if (!ctx) return GSQL_E_INVALID;
    GSQL_CUDA(ctx, cudaStreamSynchronize(ctx->stream));
    if (ctx->own_stream) cudaStreamDestroy(ctx->stream);
    ctx->stream = (cudaStream_t)s;
    ctx->own_stream = false;
    return GSQL_OK;
}

extern "C" int64_t gsql_ctx_launch_count(const gsql_ctx *ctx) { return ctx ? ctx->launches : 0; }

// ------------------------------------------------------------------------------------------------ profiling
static cudaEvent_t take_event(gsql_ctx *ctx) {
    if (!ctx->event_pool.empty()) {
        cudaEvent_t e = ctx->event_pool.back();
        ctx->event_pool.pop_back();
        return e;
    }
    cudaEvent_t e;
    cudaEventCreate(&e);
    return e;
}

KernelScope::KernelScope(gsql_ctx *c, const char *name, cudaStream_t on) : ctx(c), stream(on ? on : c->stream) {
    c->launches++;
    if (!c->profiling) return;
    for (size_t i = 0; i < c->prof.size(); i++)
        if (c->prof[i].name == name) { idx = (int)i; break; }
    if (idx < 0) {
        c->prof.emplace_back();
        c->prof.back().name = name;
        idx = (int)c->prof.size() - 1;
    }
    start = take_event(c);
    cudaEventRecord(start, stream);
}

KernelScope::~KernelScope() {
    if (idx < 0) return;
    cudaEvent_t stop = take_event(ctx);
    cudaEventRecord(stop, stream);
    ctx->prof[idx].pending.emplace_back(start, stop);
    ctx->prof[idx].launches++;
}

static void prof_resolve(gsql_ctx *ctx) {
    cudaStreamSynchronize(ctx->stream);
    for (auto &p : ctx->prof) {
        for (auto &ev : p.pending) {
            float ms = 0;
            cudaEventSynchronize(ev.second);  // kernels of an exchange run on its own stream
            if (cudaEventElapsedTime(&ms, ev.first, ev.second) == cudaSuccess) p.ms += ms;
            ctx->event_pool.push_back(ev.first);
            ctx->event_pool.push_back(ev.second);
        }
        p.pending.clear();
    }
}

extern "C" gsql_status gsql_ctx_profile(gsql_ctx *ctx, int enable) {
    if (!ctx) return GSQL_E_INVALID;
    prof_resolve(ctx);
    ctx->profiling = enable != 0;
    return GSQL_OK;
}

extern "C" gsql_status gsql_ctx_profile_reset(gsql_ctx *ctx) {
    if (!ctx) return GSQL_E_INVALID;
    prof_resolve(ctx);
    for (auto &p : ctx->prof) { p.launches = 0; p.ms = 0; }
    return GSQL_OK;
}

extern "C" gsql_status gsql_ctx_profile_get(gsql_ctx *ctx, const char *name, int64_t *launches, double *total_ms) {
    if (!ctx || !name) return GSQL_E_INVALID;
    prof_resolve(ctx);
    if (launches) *launches = 0;
    if (total_ms) *total_ms = 0;
    for (auto &p : ctx->prof)
        if (p.name == name) {
            if (launches) *launches = p.launches;
            if (total_ms) *total_ms = p.ms;
        }
    return GSQL_OK;
}

extern "C" int gsql_ctx_profile_dump(gsql_ctx *ctx, char *buf, size_t cap) {
    if (!ctx) return 0;
    prof_resolve(ctx);
    size_t off = 0;
    int n = 0;
    for (auto &p : ctx->prof) {
        if (p.launches == 0) continue;
        int w = snprintf(buf + off, off < cap ? cap - off : 0, "%s %lld %.6f\n", p.name.c_str(), (long long)p.launches, p.ms);
        if (w > 0) off += (size_t)w;
        n++;
    }
    return n;
}

// ------------------------------------------------------------------------------------------------ memory
gsql_status dev_alloc(gsql_ctx *ctx, size_t bytes, void **out) {
    if (bytes == 0) bytes = 16;
    cudaError_t e = cudaMallocAsync(out, bytes, ctx->stream);
    if (e != cudaSuccess) {
        cudaGetLastError();
        return gsql_set_error(ctx, GSQL_E_OOM, "cudaMallocAsync(%zu bytes): %s", bytes, cudaGetErrorString(e));
    }
    return GSQL_OK;
}

void dev_free(gsql_ctx *ctx, void *p) {
    if (p) cudaFreeAsync(p, ctx->stream);
}

extern "C" gsql_status gsql_host_alloc(size_t bytes, void **out) {
    if (!out) return GSQL_E_INVALID;
    return cudaHostAlloc(out, bytes ? bytes : 16, cudaHostAllocDefault) == cudaSuccess ? GSQL_OK : GSQL_E_OOM;
}
extern "C" void gsql_host_free(void *p) {
    if (p) cudaFreeHost(p);
}
extern "C" gsql_status gsql_device_alloc(gsql_ctx *ctx, size_t bytes, void **out) {
    if (!ctx || !out) return GSQL_E_INVALID;
    return dev_alloc(ctx, bytes, out);
}
extern "C" void gsql_device_free(gsql_ctx *ctx, void *p) {
    if (ctx) dev_free(ctx, p);
}
extern "C" gsql_status gsql_memcpy_h2d(gsql_ctx *ctx, void *dst, const void *src, size_t bytes) {
    if (!ctx) return GSQL_E_INVALID;
    GSQL_CUDA(ctx, cudaMemcpyAsync(dst, src, bytes, cudaMemcpyHostToDevice, ctx->stream));
    return GSQL_OK;
}
extern "C" gsql_status gsql_memcpy_d2h(gsql_ctx *ctx, void *dst, const void *src, size_t bytes) {
    if (!ctx) return GSQL_E_INVALID;
    GSQL_CUDA(ctx, cudaMemcpyAsync(dst, src, bytes, cudaMemcpyDeviceToHost, ctx->stream));
    GSQL_CUDA(ctx, cudaStreamSynchronize(ctx->stream));
    return GSQL_OK;
}

gsql_status validate_batch(gsql_ctx *ctx, const gsql_batch *b, int32_t expect_cols, const int32_t *expect_types) {
    if (!b || b->rows < 0 || b->ncols < 0 || b->ncols > GSQL_MAX_COLS || (b->ncols > 0 && !b->cols))
        return gsql_set_error(ctx, GSQL_E_INVALID, "malformed batch");
    if (b->mem != GSQL_MEM_HOST && b->mem != GSQL_MEM_DEVICE) return gsql_set_error(ctx, GSQL_E_INVALID, "bad batch.mem");
    if (expect_cols >= 0 && b->ncols != expect_cols)
        return gsql_set_error(ctx, GSQL_E_INVALID, "batch has %d columns, expected %d", b->ncols, expect_cols);
    for (int i = 0; i < b->ncols; i++) {
        int t = b->cols[i].type;
        if (t != GSQL_T_INT32 && t != GSQL_T_INT64 && t != GSQL_T_FP64 && t != GSQL_T_DEC128)
            return gsql_set_error(ctx, GSQL_E_INVALID, "column %d: unknown type %d", i, t);
        if (expect_types && t != expect_types[i])
            return gsql_set_error(ctx, GSQL_E_INVALID, "column %d: type %d, expected %d", i, t, expect_types[i]);
        if (b->rows > 0 && !b->cols[i].data) return gsql_set_error(ctx, GSQL_E_INVALID, "column %d: null data", i);
    }
    return GSQL_OK;
}

gsql_status stage_batch(gsql_ctx *ctx, const gsql_batch *in, StagedBatch *out) {
    out->rows = in->rows;
    out->ncols = in->ncols;
    for (int i = 0; i < in->ncols; i++) {
        const gsql_col &c = in->cols[i];
        DCol &d = out->cols[i];
        d.type = c.type;
        d.pad = 0;
        if (in->mem == GSQL_MEM_DEVICE || in->rows == 0) {
            d.data = c.data;
            d.nulls = in->rows == 0 ? nullptr : c.nulls;
            continue;
        }
        size_t bytes = (size_t)in->rows * gsql_type_width(c.type);
        DevBuf *b = new DevBuf();
        out->owned.push_back(b);
        GSQL_TRY(b->alloc(ctx, bytes));
        GSQL_CUDA(ctx, cudaMemcpyAsync(b->p, c.data, bytes, cudaMemcpyHostToDevice, ctx->stream));
        d.data = b->p;
        d.nulls = nullptr;
        if (c.nulls) {
            DevBuf *nb = new DevBuf();
            out->owned.push_back(nb);
            GSQL_TRY(nb->alloc(ctx, (size_t)in->rows));
            GSQL_CUDA(ctx, cudaMemcpyAsync(nb->p, c.nulls, (size_t)in->rows, cudaMemcpyHostToDevice, ctx->stream));
            d.nulls = nb->as<uint8_t>();
        }
    }
    return GSQL_OK;
}

DColSet batch_cols(const gsql_batch *b) {
    DColSet s;
    memset(&s, 0, sizeof(s));
    s.n = b->ncols;
    for (int i = 0; i < b->ncols; i++) s.c[i] = DCol{b->cols[i].data, b->cols[i].nulls, b->cols[i].type, 0};
    return s;
}

// ------------------------------------------------------------------------------------------------ row store
void RowStore::init(const int32_t *t, int n) {
    ncols = n;
    for (int e = 0; e < n; e++) types[e] = t[e];
}

gsql_status RowStore::reserve(gsql_ctx *ctx, int64_t need, int64_t hint) {
    if (need <= cap) return GSQL_OK;
    int64_t c = cap ? cap : 1024;
    if (hint > c) c = hint;
    while (c < need) c *= 2;
    for (int e = 0; e < ncols; e++) {
        const size_t w = gsql_type_width(types[e]);
        GSQL_TRY(data[e].grow(ctx, (size_t)c * w, (size_t)rows * w));
        if (has_nulls[e]) GSQL_TRY(nulls[e].grow(ctx, (size_t)c, (size_t)rows));
    }
    cap = c;
    return GSQL_OK;
}

gsql_status RowStore::make_room(gsql_ctx *ctx, const DColSet &src, int64_t n) {
    GSQL_TRY(reserve(ctx, rows + n));
    for (int e = 0; e < ncols; e++) {
        if (!src.c[e].nulls || has_nulls[e]) continue;
        GSQL_TRY(nulls[e].alloc(ctx, (size_t)cap));
        GSQL_CUDA(ctx, cudaMemsetAsync(nulls[e].p, 0, (size_t)rows, ctx->stream));
        has_nulls[e] = true;
    }
    return GSQL_OK;
}

gsql_status RowStore::append(gsql_ctx *ctx, const DColSet &src, int64_t n, cudaMemcpyKind kind) {
    GSQL_TRY(make_room(ctx, src, n));
    for (int e = 0; e < ncols; e++) {
        const size_t w = gsql_type_width(types[e]);
        GSQL_CUDA(ctx, cudaMemcpyAsync(data[e].as<char>() + (size_t)rows * w, src.c[e].data, (size_t)n * w, kind, ctx->stream));
        if (src.c[e].nulls) GSQL_CUDA(ctx, cudaMemcpyAsync(nulls[e].as<uint8_t>() + rows, src.c[e].nulls, (size_t)n, kind, ctx->stream));
        else if (has_nulls[e]) GSQL_CUDA(ctx, cudaMemsetAsync(nulls[e].as<uint8_t>() + rows, 0, (size_t)n, ctx->stream));
    }
    rows += n;
    return GSQL_OK;
}

DColSet RowStore::view() const {
    DColSet s;
    memset(&s, 0, sizeof(s));
    s.n = ncols;
    for (int e = 0; e < ncols; e++) s.c[e] = DCol{data[e].p, has_nulls[e] ? nulls[e].as<uint8_t>() : nullptr, types[e], 0};
    return s;
}

size_t RowStore::bytes() const {
    size_t b = 0;
    for (int e = 0; e < ncols; e++) b += data[e].bytes + nulls[e].bytes;
    return b;
}

gsql_status out_bind(gsql_ctx *ctx, const gsql_batch *out, int64_t rows, OutBinding *b) {
    for (int c = 0; c < out->ncols; c++) {
        const gsql_col &col = out->cols[c];
        if (out->mem == GSQL_MEM_DEVICE) {
            b->data[c] = col.data;
            b->nulls[c] = col.nulls;
            continue;
        }
        GSQL_TRY(b->scratch[c].alloc(ctx, (size_t)rows * gsql_type_width(col.type)));
        b->data[c] = b->scratch[c].p;
        if (col.nulls) {
            GSQL_TRY(b->scratch_nulls[c].alloc(ctx, (size_t)rows));
            b->nulls[c] = b->scratch_nulls[c].as<uint8_t>();
        }
    }
    return GSQL_OK;
}

gsql_status out_download(gsql_ctx *ctx, gsql_batch *out, int64_t rows, const OutBinding &b) {
    if (out->mem == GSQL_MEM_DEVICE || rows == 0) return GSQL_OK;
    for (int c = 0; c < out->ncols; c++) {
        const gsql_col &col = out->cols[c];
        GSQL_CUDA(ctx, cudaMemcpyAsync(col.data, b.data[c], (size_t)rows * gsql_type_width(col.type), cudaMemcpyDeviceToHost, ctx->stream));
        if (col.nulls) GSQL_CUDA(ctx, cudaMemcpyAsync(col.nulls, b.nulls[c], (size_t)rows, cudaMemcpyDeviceToHost, ctx->stream));
    }
    GSQL_CUDA(ctx, cudaStreamSynchronize(ctx->stream));
    return GSQL_OK;
}

gsql_status out_copy_rows(gsql_ctx *ctx, gsql_batch *out, int c, int64_t dst_row, const DevBuf &data, const DevBuf &nulls, int64_t src_row,
                          int64_t n) {
    const gsql_col &col = out->cols[c];
    const size_t w = (size_t)gsql_type_width(col.type);
    const cudaMemcpyKind kind = out->mem == GSQL_MEM_DEVICE ? cudaMemcpyDeviceToDevice : cudaMemcpyDeviceToHost;
    GSQL_CUDA(ctx, cudaMemcpyAsync((char *)col.data + (size_t)dst_row * w, data.as<char>() + (size_t)src_row * w, (size_t)n * w, kind, ctx->stream));
    GSQL_CUDA(ctx, cudaMemcpyAsync(col.nulls + dst_row, nulls.as<uint8_t>() + src_row, (size_t)n, kind, ctx->stream));
    return GSQL_OK;
}

// ------------------------------------------------------------------------------------------------ null masks
struct MaskSet {
    const uint8_t *m[GSQL_MAX_COLS];
    int32_t n;
};
__global__ void __launch_bounds__(256) k_any_null(const __grid_constant__ MaskSet M, int64_t rows, int32_t *__restrict__ any) {
    for (int c = 0; c < M.n; c++) {
        const uint8_t *m = M.m[c];
        if (!m) continue;
        // head bytes up to 16-byte alignment, 16-byte body, tail
        const int64_t head = ((16 - ((uintptr_t)m & 15)) & 15) < rows ? (int64_t)((16 - ((uintptr_t)m & 15)) & 15) : rows;
        const int64_t body = (rows - head) / 16;
        const int4 *b = reinterpret_cast<const int4 *>(m + head);
        int acc = 0;
        for (int64_t i = blockIdx.x * (int64_t)blockDim.x + threadIdx.x; i < body; i += (int64_t)gridDim.x * blockDim.x) {
            int4 v = __ldg(b + i);
            acc |= v.x | v.y | v.z | v.w;
        }
        if (blockIdx.x == 0) {
            for (int64_t i = threadIdx.x; i < head; i += blockDim.x) acc |= m[i];
            for (int64_t i = head + body * 16 + threadIdx.x; i < rows; i += blockDim.x) acc |= m[i];
        }
        if (__any_sync(0xffffffffu, acc != 0) && (threadIdx.x & 31) == 0) any[c] = 1;
    }
}

gsql_status masks_any_null(gsql_ctx *ctx, int n, const uint8_t *const *masks, int64_t rows, int mem, bool *any) {
    bool some = false;
    for (int i = 0; i < n; i++) { any[i] = false; some |= masks[i] != nullptr; }
    if (!some || rows == 0) return GSQL_OK;
    if (mem == GSQL_MEM_HOST) {
        for (int i = 0; i < n; i++) {
            const uint8_t *m = masks[i];
            if (!m) continue;
            int64_t r = 0;
            for (; r < rows && ((uintptr_t)(m + r) & 7); r++) if (m[r]) { any[i] = true; break; }
            if (any[i]) continue;
            const uint64_t *w = reinterpret_cast<const uint64_t *>(m + r);
            const int64_t nw = (rows - r) / 8;
            uint64_t acc = 0;
            for (int64_t k = 0; k < nw && !acc; k += 512) {
                const int64_t e = k + 512 < nw ? k + 512 : nw;
                for (int64_t q = k; q < e; q++) acc |= w[q];
            }
            if (acc) { any[i] = true; continue; }
            for (r += nw * 8; r < rows; r++) if (m[r]) { any[i] = true; break; }
        }
        return GSQL_OK;
    }
    MaskSet M;
    memset(&M, 0, sizeof(M));
    M.n = n;
    for (int i = 0; i < n; i++) M.m[i] = masks[i];
    DevBuf flags;
    GSQL_TRY(flags.alloc(ctx, (size_t)GSQL_MAX_COLS * 4));
    GSQL_CUDA(ctx, cudaMemsetAsync(flags.p, 0, (size_t)GSQL_MAX_COLS * 4, ctx->stream));
    {
        KernelScope ks(ctx, "any_null");
        int64_t g = div_up(rows / 16 + 1, 256);
        if (g > (int64_t)ctx->sm_count * 8) g = (int64_t)ctx->sm_count * 8;
        k_any_null<<<(int)g, 256, 0, ctx->stream>>>(M, rows, flags.as<int32_t>());
    }
    GSQL_CUDA(ctx, cudaGetLastError());
    int32_t h[GSQL_MAX_COLS];
    GSQL_CUDA(ctx, cudaMemcpyAsync(h, flags.p, (size_t)n * 4, cudaMemcpyDeviceToHost, ctx->stream));
    GSQL_CUDA(ctx, cudaStreamSynchronize(ctx->stream));
    for (int i = 0; i < n; i++) any[i] = h[i] != 0;
    return GSQL_OK;
}

gsql_status strip_zero_masks(gsql_ctx *ctx, const gsql_batch *in, gsql_batch *out, gsql_col *cols_storage) {
    *out = *in;
    out->cols = cols_storage;
    const uint8_t *masks[GSQL_MAX_COLS];
    bool any[GSQL_MAX_COLS];
    for (int i = 0; i < in->ncols; i++) {
        cols_storage[i] = in->cols[i];
        masks[i] = in->cols[i].nulls;
    }
    GSQL_TRY(masks_any_null(ctx, in->ncols, masks, in->rows, in->mem, any));
    for (int i = 0; i < in->ncols; i++)
        if (!any[i]) cols_storage[i].nulls = nullptr;
    return GSQL_OK;
}

// ------------------------------------------------------------------------------------------------ hashing
__global__ void __launch_bounds__(256) k_hash_rows(KeySet ks, int64_t rows, int32_t *__restrict__ out) {
    for (int64_t r = blockIdx.x * (int64_t)blockDim.x + threadIdx.x; r < rows; r += (int64_t)gridDim.x * blockDim.x)
        out[r] = gsql_row_hash(ks, r);
}

__global__ void __launch_bounds__(256)
    k_partition_ids(const int32_t *__restrict__ hash, int64_t rows, int32_t nparts, bool pow2, int32_t *__restrict__ out) {
    for (int64_t r = blockIdx.x * (int64_t)blockDim.x + threadIdx.x; r < rows; r += (int64_t)gridDim.x * blockDim.x)
        out[r] = gsql_partition_of(hash[r], nparts, pow2);
}

extern "C" gsql_status gsql_hash_rows(gsql_ctx *ctx, const gsql_batch *batch, const int32_t *key_cols, int32_t nkeys,
                                      const int32_t *unified_types, int32_t *out) {
    if (!ctx) return GSQL_E_INVALID;
    if (ctx->sticky) return GSQL_E_CUDA;
    GSQL_TRY(validate_batch(ctx, batch, -1, nullptr));
    if (nkeys < 0 || nkeys > GSQL_MAX_KEYS || (batch->rows > 0 && !out)) return gsql_set_error(ctx, GSQL_E_INVALID, "bad keys/out");
    if (batch->rows == 0) return GSQL_OK;
    StagedBatch sb;
    GSQL_TRY(stage_batch(ctx, batch, &sb));
    KeySet ks;
    ks.n = nkeys;
    for (int i = 0; i < nkeys; i++) {
        if (key_cols[i] < 0 || key_cols[i] >= batch->ncols) return gsql_set_error(ctx, GSQL_E_INVALID, "key col out of range");
        ks.c[i] = sb.cols[key_cols[i]];
        ks.utype[i] = unified_types ? unified_types[i] : sb.cols[key_cols[i]].type;
    }
    DevBuf dout;
    int32_t *d_out = out;
    if (batch->mem == GSQL_MEM_HOST) {
        GSQL_TRY(dout.alloc(ctx, (size_t)batch->rows * 4));
        d_out = dout.as<int32_t>();
    }
    {
        KernelScope ks_(ctx, "hash_rows");
        k_hash_rows<<<grid_for(ctx, batch->rows, 256, 16), 256, 0, ctx->stream>>>(ks, batch->rows, d_out);
    }
    GSQL_CUDA(ctx, cudaGetLastError());
    if (batch->mem == GSQL_MEM_HOST) {
        GSQL_CUDA(ctx, cudaMemcpyAsync(out, d_out, (size_t)batch->rows * 4, cudaMemcpyDeviceToHost, ctx->stream));
        GSQL_CUDA(ctx, cudaStreamSynchronize(ctx->stream));
    }
    return GSQL_OK;
}

extern "C" gsql_status gsql_partition_ids(gsql_ctx *ctx, const int32_t *hash, int64_t rows, int32_t nparts, int32_t *out,
                                          int32_t mem) {
    if (!ctx) return GSQL_E_INVALID;
    if (ctx->sticky) return GSQL_E_CUDA;
    if (rows < 0 || nparts <= 0 || (rows > 0 && (!hash || !out))) return gsql_set_error(ctx, GSQL_E_INVALID, "bad args");
    if (rows == 0) return GSQL_OK;
    DevBuf din, dout;
    const int32_t *d_in = hash;
    int32_t *d_out = out;
    if (mem == GSQL_MEM_HOST) {
        GSQL_TRY(din.alloc(ctx, (size_t)rows * 4));
        GSQL_TRY(dout.alloc(ctx, (size_t)rows * 4));
        GSQL_CUDA(ctx, cudaMemcpyAsync(din.p, hash, (size_t)rows * 4, cudaMemcpyHostToDevice, ctx->stream));
        d_in = din.as<int32_t>();
        d_out = dout.as<int32_t>();
    }
    bool pow2 = (nparts & -nparts) == nparts;
    {
        KernelScope ks_(ctx, "partition_ids");
        k_partition_ids<<<grid_for(ctx, rows, 256, 16), 256, 0, ctx->stream>>>(d_in, rows, nparts, pow2, d_out);
    }
    GSQL_CUDA(ctx, cudaGetLastError());
    if (mem == GSQL_MEM_HOST) {
        GSQL_CUDA(ctx, cudaMemcpyAsync(out, d_out, (size_t)rows * 4, cudaMemcpyDeviceToHost, ctx->stream));
        GSQL_CUDA(ctx, cudaStreamSynchronize(ctx->stream));
    }
    return GSQL_OK;
}
