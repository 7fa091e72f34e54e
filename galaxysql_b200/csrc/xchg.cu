// xchg.cu — hash-partition exchange behind gsql_xchg_* and gsql_comm_*.
//
// Reference path replaced (EX/ = polardbx-executor/src/main/java/com/alibaba/polardbx/executor/):
//   local : EX/mpp/operator/PartitioningExchanger.java:71-135 (consumeChunk: per-row partition id, per-destination
//           chunk build), HashBucketFunction (PartitionedOutputCollector.java:282-302)
//   remote: EX/mpp/operator/PartitionedOutputCollector.java:170-196 (partitionPage) + HashPartitionFunction:253-279,
//           PagesSerde / PartitionedOutputBuffer / ExchangeClient HTTP pull (ExchangeClient.java:62-548)
// Destination ids are bit-exact with ExecUtils.partition(Chunk.hashCode) so GPU and stock Java tasks route the
// same row to the same consumer.
//
// Shape: histogram (keys only) -> exclusive scan over [partition][block] -> scatter of all columns into one
// buffer whose partitions are contiguous; across GPUs the contiguous segments are exchanged with one grouped
// ncclSend/ncclRecv AllToAllv per column over NVLink / NVSwitch — no serialisation, no compression.
// NCCL is bound at run time (dlopen) so that the library shares the process's NCCL with torch.distributed.
#include <dlfcn.h>
#include <nccl.h>
#include <stdlib.h>

#include <cub/device/device_scan.cuh>

#include "common.cuh"

namespace {

constexpr int XBLOCK = 256;

struct XParams {
    DColSet in;
    KeySet keys;
    int32_t nparts, pow2;
    int64_t rows, chunk;  // rows per block
    int32_t nblocks, mode;
    int64_t row_base;     // index of row 0 inside the caller's batch (round-robin destinations continue across slabs)
};

struct XOut {
    void *data[GSQL_MAX_COLS];
    uint8_t *nulls[GSQL_MAX_COLS];
};

__device__ __forceinline__ int row_part(const XParams &P, int64_t r) {
    if (P.mode == GSQL_XCHG_RANDOM) return (int)((unsigned long long)(P.row_base + r) % (unsigned)P.nparts);  // RandomExchanger: balance only
    return gsql_partition_of(gsql_row_hash(P.keys, r), P.nparts, P.pow2 != 0);
}

// hist[p * nblocks + b] = rows of block b's chunk routed to p
__global__ void __launch_bounds__(XBLOCK) k_xchg_hist(const __grid_constant__ XParams P, int64_t *__restrict__ hist) {
    extern __shared__ unsigned int sh[];
    for (int i = threadIdx.x; i < P.nparts; i += XBLOCK) sh[i] = 0;
    __syncthreads();
    int64_t r0 = (int64_t)blockIdx.x * P.chunk;
    int64_t r1 = r0 + P.chunk < P.rows ? r0 + P.chunk : P.rows;
    for (int64_t r = r0 + threadIdx.x; r < r1; r += XBLOCK) atomicAdd(&sh[row_part(P, r)], 1u);
    __syncthreads();
    for (int i = threadIdx.x; i < P.nparts; i += XBLOCK) hist[(int64_t)i * P.nblocks + blockIdx.x] = sh[i];
}

__global__ void __launch_bounds__(XBLOCK)
    k_xchg_scatter(const __grid_constant__ XParams P, const int64_t *__restrict__ offs, const __grid_constant__ XOut O) {
    extern __shared__ unsigned long long cur[];
    for (int i = threadIdx.x; i < P.nparts; i += XBLOCK) cur[i] = (unsigned long long)offs[(int64_t)i * P.nblocks + blockIdx.x];
    __syncthreads();
    int64_t r0 = (int64_t)blockIdx.x * P.chunk;
    int64_t r1 = r0 + P.chunk < P.rows ? r0 + P.chunk : P.rows;
    for (int64_t base = r0; base < r1; base += XBLOCK) {
        int64_t r = base + threadIdx.x;
        bool live = r < r1;
        int p = live ? row_part(P, r) : -1;
        // warp-aggregated cursor bump: one shared-memory atomic per distinct destination per warp
        unsigned peers = __match_any_sync(0xffffffffu, p);
        int lane = threadIdx.x & 31;
        int leader = __ffs(peers) - 1;
        unsigned long long basepos = 0;
        if (live && lane == leader) basepos = atomicAdd(&cur[p], (unsigned long long)__popc(peers));
        basepos = __shfl_sync(0xffffffffu, basepos, leader);
        if (!live) continue;
        int64_t pos = (int64_t)basepos + __popc(peers & ((1u << lane) - 1));
        for (int c = 0; c < P.in.n; c++) {
            const DCol &col = P.in.c[c];
            if (col.type == GSQL_T_INT32) reinterpret_cast<int32_t *>(O.data[c])[pos] = reinterpret_cast<const int32_t *>(col.data)[r];
            else reinterpret_cast<int64_t *>(O.data[c])[pos] = reinterpret_cast<const int64_t *>(col.data)[r];
            if (O.nulls[c]) O.nulls[c][pos] = col.nulls ? col.nulls[r] : 0;
        }
    }
}

// ------------------------------------------------------------------------------------------------ NCCL binding
struct NcclApi {
    void *handle = nullptr;
    ncclResult_t (*GetUniqueId)(ncclUniqueId *) = nullptr;
    ncclResult_t (*CommInitRank)(ncclComm_t *, int, ncclUniqueId, int) = nullptr;
    ncclResult_t (*CommDestroy)(ncclComm_t) = nullptr;
    ncclResult_t (*CommSplit)(ncclComm_t, int, int, ncclComm_t *, ncclConfig_t *) = nullptr;
    ncclResult_t (*AllGather)(const void *, void *, size_t, ncclDataType_t, ncclComm_t, cudaStream_t) = nullptr;
    ncclResult_t (*Send)(const void *, size_t, ncclDataType_t, int, ncclComm_t, cudaStream_t) = nullptr;
    ncclResult_t (*Recv)(void *, size_t, ncclDataType_t, int, ncclComm_t, cudaStream_t) = nullptr;
    ncclResult_t (*GroupStart)() = nullptr;
    ncclResult_t (*GroupEnd)() = nullptr;
    const char *(*GetErrorString)(ncclResult_t) = nullptr;
    bool ok = false;
};

NcclApi *nccl_api() {
    static NcclApi api;
    static bool tried = false;
    if (tried) return &api;
    tried = true;
    // Prefer the NCCL already in the process (torch's bundled one), else the system library.
    void *h = dlopen("libnccl.so.2", RTLD_NOW | RTLD_NOLOAD | RTLD_GLOBAL);
    if (!h) h = dlopen("libnccl.so.2", RTLD_NOW | RTLD_GLOBAL);
    if (!h) h = dlopen("libnccl.so", RTLD_NOW | RTLD_GLOBAL);
    if (!h) return &api;
    api.handle = h;
#define BIND(field, sym) *(void **)(&api.field) = dlsym(h, sym)
    BIND(GetUniqueId, "ncclGetUniqueId");
    BIND(CommInitRank, "ncclCommInitRank");
    BIND(CommDestroy, "ncclCommDestroy");
    BIND(CommSplit, "ncclCommSplit");
    BIND(AllGather, "ncclAllGather");
    BIND(Send, "ncclSend");
    BIND(Recv, "ncclRecv");
    BIND(GroupStart, "ncclGroupStart");
    BIND(GroupEnd, "ncclGroupEnd");
    BIND(GetErrorString, "ncclGetErrorString");
#undef BIND
    api.ok = api.GetUniqueId && api.CommInitRank && api.CommDestroy && api.AllGather && api.Send && api.Recv && api.GroupStart &&
             api.GroupEnd && api.GetErrorString;
    return &api;
}

#define GSQL_NCCL(ctx, call)                                                                                            \
    do {                                                                                                                \
        ncclResult_t _r = (call);                                                                                       \
        if (_r != ncclSuccess) {                                                                                        \
            (ctx)->sticky = true;                                                                                       \
            return gsql_set_error((ctx), GSQL_E_NCCL, "%s:%d %s -> %s", __FILE__, __LINE__, #call, nccl_api()->GetErrorString(_r)); \
        }                                                                                                               \
    } while (0)

int grid_rows(gsql_ctx *ctx, int64_t rows, int block, int per_sm) {
    int64_t g = div_up(rows, block);
    int64_t cap = (int64_t)ctx->sm_count * per_sm;
    if (g > cap) g = cap;
    if (g < 1) g = 1;
    return (int)g;
}

}  // namespace

struct P2PCtrl;

struct gsql_xchg {
    gsql_ctx *ctx;
    gsql_xchg_spec spec;
    // send staging of the NCCL shuffle (partition-ordered columns), kept across calls: a shuffle of N rows stages N rows,
    // and re-allocating those gigabytes on every call raced the stream-ordered frees of the previous one
    DevBuf sdata[GSQL_MAX_COLS], snull[GSQL_MAX_COLS];
    // ---- partition-and-push over peer memory (gsql_xchg_open_p2p)
    bool p2p = false;
    char *base = nullptr;                       // this rank's allocation: control block, then the receive columns
    char *peer_base[GSQL_MAX_RANKS] = {nullptr};  // the same allocation of every rank, mapped here (CUDA IPC); [rank] = base
    size_t alloc_bytes = 0;
    int64_t cap = 0;
    int64_t col_off[GSQL_MAX_COLS], null_off[GSQL_MAX_COLS];
    cudaStream_t pstream = nullptr;             // pushes and their barriers run here, beside the context stream
    cudaEvent_t in_ev = nullptr, slab_ev[GSQL_MAX_SLABS] = {nullptr};
    unsigned long long seq = 0;                 // barrier sequence number (identical on all ranks: calls are collective)
    int64_t pushes = 0;
    int32_t last_slabs = 0;
    int64_t slab_rows[GSQL_MAX_SLABS], slab_base[GSQL_MAX_SLABS];
    DevBuf hist[GSQL_MAX_SLABS], offs[GSQL_MAX_SLABS], scan_tmp;
    long long *host_matrix = nullptr;           // pinned: counts[src][slab][dst] of the current push
    int32_t *host_err = nullptr;                // pinned copy of the control block's error word
};

extern "C" gsql_status gsql_xchg_create(gsql_ctx *ctx, const gsql_xchg_spec *spec, gsql_xchg **out) {
    if (!ctx || !spec || !out) return GSQL_E_INVALID;
    *out = nullptr;
    const gsql_xchg_spec &s = *spec;
    if (s.n_cols < 1 || s.n_cols > GSQL_MAX_COLS || s.n_channels < 0 || s.n_channels > GSQL_MAX_KEYS || s.nparts < 1 || s.nparts > GSQL_MAX_PARTS ||
        s.mode < GSQL_XCHG_HASH || s.mode > GSQL_XCHG_RANDOM)
        return gsql_set_error(ctx, GSQL_E_INVALID, "bad exchange spec");
    for (int i = 0; i < s.n_cols; i++)
        if (s.types[i] < GSQL_T_INT32 || s.types[i] > GSQL_T_FP64) return gsql_set_error(ctx, GSQL_E_UNSUPPORTED, "column %d type", i);
    for (int i = 0; i < s.n_channels; i++)
        if (s.channels[i] < 0 || s.channels[i] >= s.n_cols || s.key_types[i] < GSQL_T_INT32 || s.key_types[i] > GSQL_T_FP64)
            return gsql_set_error(ctx, GSQL_E_INVALID, "channel %d", i);
    gsql_xchg *x = new gsql_xchg();
    x->ctx = ctx;
    gsql_ctx_retain(ctx);
    x->spec = s;
    *out = x;
    return GSQL_OK;
}

static void p2p_close(gsql_xchg *x);

extern "C" void gsql_xchg_destroy(gsql_xchg *x) {
    if (!x) return;
    gsql_ctx *ctx = x->ctx;
    cudaSetDevice(ctx->device);
    p2p_close(x);
    delete x;
    if (!ctx->sticky) cudaStreamSynchronize(ctx->stream);  // stream-ordered frees have really happened (see gsql_join_destroy)
    gsql_ctx_release(ctx);
}

// Partitions staged device columns into `O` (device).  d_part_offsets receives nparts+1 int64 offsets (device).
static gsql_status partition_device(gsql_xchg *x, const StagedBatch &sb, const XOut &O, DevBuf *offs_out, int64_t *host_counts) {
    gsql_ctx *ctx = x->ctx;
    const gsql_xchg_spec &s = x->spec;
    XParams P;
    memset(&P, 0, sizeof(P));
    P.in.n = sb.ncols;
    for (int i = 0; i < sb.ncols; i++) P.in.c[i] = sb.cols[i];
    P.keys.n = s.n_channels;
    for (int i = 0; i < s.n_channels; i++) {
        P.keys.c[i] = sb.cols[s.channels[i]];
        P.keys.utype[i] = s.key_types[i];
    }
    P.nparts = s.nparts;
    P.pow2 = (s.nparts & -s.nparts) == s.nparts;
    P.mode = s.mode;
    P.rows = sb.rows;
    int nblocks = grid_rows(ctx, sb.rows, 4096, 8);
    P.chunk = div_up(sb.rows, nblocks);
    P.chunk = div_up(P.chunk, XBLOCK) * XBLOCK;
    nblocks = (int)div_up(sb.rows, P.chunk);
    if (nblocks < 1) nblocks = 1;
    P.nblocks = nblocks;
    int64_t nh = (int64_t)s.nparts * nblocks;
    DevBuf hist, tmp;
    GSQL_TRY(hist.alloc(ctx, (size_t)(nh + 1) * 8));
    GSQL_TRY(offs_out->alloc(ctx, (size_t)(nh + 1) * 8));
    GSQL_CUDA(ctx, cudaMemsetAsync((char *)hist.p + nh * 8, 0, 8, ctx->stream));
    {
        KernelScope ks(ctx, "xchg_hist");
        k_xchg_hist<<<nblocks, XBLOCK, s.nparts * sizeof(unsigned int), ctx->stream>>>(P, hist.as<int64_t>());
    }
    GSQL_CUDA(ctx, cudaGetLastError());
    size_t tb = 0;
    GSQL_CUDA(ctx, cub::DeviceScan::ExclusiveSum(nullptr, tb, hist.as<int64_t>(), offs_out->as<int64_t>(), nh + 1, ctx->stream));
    GSQL_TRY(tmp.alloc(ctx, tb));
    {
        KernelScope ks(ctx, "xchg_scan");
        GSQL_CUDA(ctx, cub::DeviceScan::ExclusiveSum(tmp.p, tb, hist.as<int64_t>(), offs_out->as<int64_t>(), nh + 1, ctx->stream));
    }
    {
        KernelScope ks(ctx, "xchg_scatter");
        k_xchg_scatter<<<nblocks, XBLOCK, s.nparts * sizeof(unsigned long long), ctx->stream>>>(P, offs_out->as<int64_t>(), O);
    }
    GSQL_CUDA(ctx, cudaGetLastError());
    if (host_counts) {  // partition p starts at offs[p * nblocks]
        std::vector<int64_t> starts((size_t)s.nparts + 1);
        GSQL_CUDA(ctx, cudaMemcpy2DAsync(starts.data(), 8, offs_out->p, (size_t)nblocks * 8, 8, (size_t)s.nparts, cudaMemcpyDeviceToHost, ctx->stream));
        GSQL_CUDA(ctx, cudaStreamSynchronize(ctx->stream));
        starts[(size_t)s.nparts] = sb.rows;
        for (int p = 0; p < s.nparts; p++) host_counts[p] = starts[(size_t)p + 1] - starts[(size_t)p];
    }
    return GSQL_OK;
}

extern "C" gsql_status gsql_xchg_partition(gsql_xchg *x, const gsql_batch *in, gsql_batch *out, int64_t *part_counts) {
    if (!x || !in || !out || !part_counts) return GSQL_E_INVALID;
    gsql_ctx *ctx = x->ctx;
    if (ctx->sticky) return GSQL_E_CUDA;
    const gsql_xchg_spec &s = x->spec;
    GSQL_TRY(validate_batch(ctx, in, s.n_cols, s.types));
    GSQL_TRY(validate_batch(ctx, out, s.n_cols, s.types));
    if (in->mem != out->mem) return gsql_set_error(ctx, GSQL_E_INVALID, "in and out must live in the same memory space");
    if (s.mode == GSQL_XCHG_BROADCAST) return gsql_set_error(ctx, GSQL_E_UNSUPPORTED, "local broadcast: the consumers of one GPU share the device batch, nothing to partition");
    for (int p = 0; p < s.nparts; p++) part_counts[p] = 0;
    out->rows = in->rows;
    if (in->rows == 0) return GSQL_OK;
    GSQL_CUDA(ctx, cudaSetDevice(ctx->device));
    for (int c = 0; c < s.n_cols; c++)
        if (in->cols[c].nulls && !out->cols[c].nulls) return gsql_set_error(ctx, GSQL_E_INVALID, "output column %d needs a nulls buffer", c);
    StagedBatch sb;
    GSQL_TRY(stage_batch(ctx, in, &sb));
    XOut O;
    memset(&O, 0, sizeof(O));
    DevBuf odata[GSQL_MAX_COLS], onull[GSQL_MAX_COLS];
    for (int c = 0; c < s.n_cols; c++) {
        if (in->mem == GSQL_MEM_DEVICE) {
            O.data[c] = out->cols[c].data;
            O.nulls[c] = out->cols[c].nulls;
        } else {
            GSQL_TRY(odata[c].alloc(ctx, (size_t)in->rows * gsql_type_width(s.types[c])));
            O.data[c] = odata[c].p;
            if (out->cols[c].nulls) {
                GSQL_TRY(onull[c].alloc(ctx, (size_t)in->rows));
                O.nulls[c] = onull[c].as<uint8_t>();
            }
        }
    }
    DevBuf offs;
    GSQL_TRY(partition_device(x, sb, O, &offs, part_counts));
    if (in->mem == GSQL_MEM_HOST) {
        for (int c = 0; c < s.n_cols; c++) {
            GSQL_CUDA(ctx, cudaMemcpyAsync(out->cols[c].data, O.data[c], (size_t)in->rows * gsql_type_width(s.types[c]), cudaMemcpyDeviceToHost, ctx->stream));
            if (out->cols[c].nulls) GSQL_CUDA(ctx, cudaMemcpyAsync(out->cols[c].nulls, O.nulls[c], (size_t)in->rows, cudaMemcpyDeviceToHost, ctx->stream));
        }
        GSQL_CUDA(ctx, cudaStreamSynchronize(ctx->stream));
    }
    return GSQL_OK;
}

// ------------------------------------------------------------------------------------------------ communicator
extern "C" gsql_status gsql_comm_unique_id(uint8_t id[128]) {
    NcclApi *api = nccl_api();
    if (!api->ok || !id) return GSQL_E_NCCL;
    ncclUniqueId uid;
    if (api->GetUniqueId(&uid) != ncclSuccess) return GSQL_E_NCCL;
    memcpy(id, uid.internal, 128);
    return GSQL_OK;
}

extern "C" gsql_status gsql_comm_init(gsql_ctx *ctx, int32_t nranks, int32_t rank, const uint8_t id[128]) {
    if (!ctx || !id || nranks < 1 || rank < 0 || rank >= nranks) return GSQL_E_INVALID;
    NcclApi *api = nccl_api();
    if (!api->ok) return gsql_set_error(ctx, GSQL_E_NCCL, "libnccl.so.2 could not be loaded");
    GSQL_CUDA(ctx, cudaSetDevice(ctx->device));
    ncclUniqueId uid;
    memcpy(uid.internal, id, 128);
    ncclComm_t comm;
    GSQL_NCCL(ctx, api->CommInitRank(&comm, nranks, uid, rank));
    ctx->nccl_comm = comm;
    ctx->nranks = nranks;
    ctx->rank = rank;
    // stripe communicators
    int want = 3;
    if (const char *e = getenv("GSQL_XCHG_STRIPES")) want = atoi(e) - 1;
    if (want > 7) want = 7;
    ctx->n_extra = 0;
    if (nranks > 1 && api->CommSplit) {
        for (int i = 0; i < want; i++) {
            ncclComm_t extra = nullptr;
            if (api->CommSplit(comm, 0, rank, &extra, nullptr) != ncclSuccess || !extra) break;
            ctx->nccl_extra[i] = extra;
            cudaStreamCreateWithFlags(&ctx->xstreams[i], cudaStreamNonBlocking);
            ctx->n_extra = i + 1;
        }
    }
    return GSQL_OK;
}

extern "C" gsql_status gsql_comm_destroy(gsql_ctx *ctx) {
    if (!ctx) return GSQL_E_INVALID;
    if (ctx->nccl_comm) {
        cudaStreamSynchronize(ctx->stream);
        for (int i = 0; i < ctx->n_extra; i++) {
            cudaStreamSynchronize(ctx->xstreams[i]);
            nccl_api()->CommDestroy((ncclComm_t)ctx->nccl_extra[i]);
            cudaStreamDestroy(ctx->xstreams[i]);
            ctx->nccl_extra[i] = nullptr;
        }
        ctx->n_extra = 0;
        nccl_api()->CommDestroy((ncclComm_t)ctx->nccl_comm);
        ctx->nccl_comm = nullptr;
    }
    return GSQL_OK;
}

// XParams of the row range [row0, row0 + rows) of a staged batch (a slab of a push).
static void fill_xparams(gsql_xchg *x, const StagedBatch &sb, int64_t row0, int64_t rows, XParams *Pp) {
    const gsql_xchg_spec &s = x->spec;
    XParams &P = *Pp;
    memset(&P, 0, sizeof(P));
    P.in.n = sb.ncols;
    for (int i = 0; i < sb.ncols; i++) {
        P.in.c[i] = sb.cols[i];
        P.in.c[i].data = (const char *)sb.cols[i].data + (size_t)row0 * gsql_type_width(sb.cols[i].type);
        if (sb.cols[i].nulls) P.in.c[i].nulls = sb.cols[i].nulls + row0;
    }
    P.keys.n = s.n_channels;
    for (int i = 0; i < s.n_channels; i++) {
        P.keys.c[i] = P.in.c[s.channels[i]];
        P.keys.utype[i] = s.key_types[i];
    }
    P.nparts = s.nparts;
    P.pow2 = (s.nparts & -s.nparts) == s.nparts;
    P.mode = s.mode;
    P.row_base = row0;
    P.rows = rows;
    int nblocks = grid_rows(x->ctx, rows, 4096, 8);
    P.chunk = div_up(rows > 0 ? rows : 1, nblocks);
    P.chunk = div_up(P.chunk, XBLOCK) * XBLOCK;
    nblocks = (int)div_up(rows, P.chunk);
    if (nblocks < 1) nblocks = 1;
    P.nblocks = nblocks;
}

extern "C" gsql_status gsql_xchg_all_to_all(gsql_xchg *x, const gsql_batch *in, gsql_batch *out, int64_t out_capacity,
                                            int64_t *out_rows, int64_t *recv_counts) {
    if (!x || !in || !out || !out_rows) return GSQL_E_INVALID;
    gsql_ctx *ctx = x->ctx;
    if (ctx->sticky) return GSQL_E_CUDA;
    const gsql_xchg_spec &s = x->spec;
    NcclApi *api = nccl_api();
    if (!ctx->nccl_comm || !api->ok) return gsql_set_error(ctx, GSQL_E_STATE, "gsql_comm_init has not been called");
    if (s.nparts != ctx->nranks) return gsql_set_error(ctx, GSQL_E_INVALID, "exchange has %d partitions but the communicator has %d ranks", s.nparts, ctx->nranks);
    if (s.mode == GSQL_XCHG_BROADCAST) return gsql_set_error(ctx, GSQL_E_UNSUPPORTED, "broadcast distribution is served by gsql_xchg_push");
    GSQL_TRY(validate_batch(ctx, in, s.n_cols, s.types));
    GSQL_TRY(validate_batch(ctx, out, s.n_cols, s.types));
    if (in->mem != GSQL_MEM_DEVICE || out->mem != GSQL_MEM_DEVICE) return gsql_set_error(ctx, GSQL_E_INVALID, "all_to_all works on device-resident batches");
    GSQL_CUDA(ctx, cudaSetDevice(ctx->device));
    const int R = ctx->nranks;
    ncclComm_t comm = (ncclComm_t)ctx->nccl_comm;
    // nullable columns must be nullable on every rank (collective shape): decided by the output buffers
    for (int c = 0; c < s.n_cols; c++)
        if (in->cols[c].nulls && !out->cols[c].nulls) return gsql_set_error(ctx, GSQL_E_INVALID, "output column %d needs a nulls buffer", c);
    // ---- 1. partition into contiguous per-destination segments
    StagedBatch sb;
    GSQL_TRY(stage_batch(ctx, in, &sb));
    XOut O;
    memset(&O, 0, sizeof(O));
    DevBuf *sdata = x->sdata, *snull = x->snull;
    int64_t srows = in->rows > 0 ? in->rows : 1;
    for (int c = 0; c < s.n_cols; c++) {
        GSQL_TRY(sdata[c].grow(ctx, (size_t)srows * gsql_type_width(s.types[c]), 0));
        O.data[c] = sdata[c].p;
        if (out->cols[c].nulls) {
            GSQL_TRY(snull[c].grow(ctx, (size_t)srows, 0));
            O.nulls[c] = snull[c].as<uint8_t>();
        }
    }
    std::vector<int64_t> send_counts((size_t)R, 0);
    DevBuf offs;
    if (in->rows > 0) GSQL_TRY(partition_device(x, sb, O, &offs, send_counts.data()));
    // ---- 2. exchange the R x R count matrix
    // every rank also publishes its receive capacity: whether ANY rank overflows is then decided identically everywhere
    // (a rank that returned E_CAPACITY on its own would leave the others blocked inside the grouped send/recv)
    DevBuf d_counts, d_matrix;
    GSQL_TRY(d_counts.alloc(ctx, (size_t)(R + 1) * 8));
    GSQL_TRY(d_matrix.alloc(ctx, (size_t)R * (R + 1) * 8));
    send_counts.push_back(out_capacity);
    GSQL_CUDA(ctx, cudaMemcpyAsync(d_counts.p, send_counts.data(), (size_t)(R + 1) * 8, cudaMemcpyHostToDevice, ctx->stream));
    GSQL_NCCL(ctx, api->AllGather(d_counts.p, d_matrix.p, (size_t)(R + 1), ncclInt64, comm, ctx->stream));
    std::vector<int64_t> wide((size_t)R * (R + 1)), matrix((size_t)R * R);
    GSQL_CUDA(ctx, cudaMemcpyAsync(wide.data(), d_matrix.p, wide.size() * 8, cudaMemcpyDeviceToHost, ctx->stream));
    GSQL_CUDA(ctx, cudaStreamSynchronize(ctx->stream));
    for (int src = 0; src < R; src++)
        for (int dst = 0; dst < R; dst++) matrix[(size_t)src * R + dst] = wide[(size_t)src * (R + 1) + dst];
    bool someone_overflows = false;
    for (int dst = 0; dst < R; dst++) {
        int64_t need = 0;
        for (int src = 0; src < R; src++) need += matrix[(size_t)src * R + dst];
        if (need > wide[(size_t)dst * (R + 1) + R]) someone_overflows = true;
    }
    int64_t total = 0;
    std::vector<int64_t> roff((size_t)R), soff((size_t)R);
    for (int src = 0; src < R; src++) {
        roff[(size_t)src] = total;
        int64_t n = matrix[(size_t)src * R + ctx->rank];
        if (recv_counts) recv_counts[src] = n;
        total += n;
    }
    int64_t acc = 0;
    for (int dst = 0; dst < R; dst++) {
        soff[(size_t)dst] = acc;
        acc += send_counts[(size_t)dst];
    }
    *out_rows = total;
    if (someone_overflows)  // on every rank alike: nobody enters the exchange
        return gsql_set_error(ctx, GSQL_E_CAPACITY, "all_to_all: a rank's receive buffer is too small (this rank needs %lld rows, capacity %lld)",
                              (long long)total, (long long)out_capacity);
    // ---- 3. AllToAllv: grouped send/recv per column (and per null mask), striped over 1 + n_extra communicators /
    //         streams so that several NCCL p2p kernels run side by side
    {
        KernelScope ks(ctx, "xchg_alltoall");
        const int K = 1 + ctx->n_extra;
        cudaEvent_t ready;
        GSQL_CUDA(ctx, cudaEventCreateWithFlags(&ready, cudaEventDisableTiming));
        GSQL_CUDA(ctx, cudaEventRecord(ready, ctx->stream));  // the partitioned send buffers are complete
        for (int k = 0; k < K; k++) {
            ncclComm_t cm = k == 0 ? comm : (ncclComm_t)ctx->nccl_extra[k - 1];
            cudaStream_t st = k == 0 ? ctx->stream : ctx->xstreams[k - 1];
            if (k > 0) GSQL_CUDA(ctx, cudaStreamWaitEvent(st, ready, 0));
            GSQL_NCCL(ctx, api->GroupStart());
            for (int c = 0; c < s.n_cols; c++) {
                size_t w = (size_t)gsql_type_width(s.types[c]);
                for (int peer = 0; peer < R; peer++) {
                    int64_t ns = send_counts[(size_t)peer], nr = matrix[(size_t)peer * R + ctx->rank];
                    // stripe k carries rows [n*k/K, n*(k+1)/K) of every segment
                    int64_t s0 = ns * k / K, s1 = ns * (k + 1) / K, r0 = nr * k / K, r1 = nr * (k + 1) / K;
                    if (s1 > s0) GSQL_NCCL(ctx, api->Send((char *)sdata[c].p + (size_t)(soff[(size_t)peer] + s0) * w, (size_t)(s1 - s0) * w, ncclInt8, peer, cm, st));
                    if (r1 > r0) GSQL_NCCL(ctx, api->Recv((char *)out->cols[c].data + (size_t)(roff[(size_t)peer] + r0) * w, (size_t)(r1 - r0) * w, ncclInt8, peer, cm, st));
                    if (out->cols[c].nulls) {
                        if (s1 > s0) GSQL_NCCL(ctx, api->Send((char *)snull[c].p + soff[(size_t)peer] + s0, (size_t)(s1 - s0), ncclInt8, peer, cm, st));
                        if (r1 > r0) GSQL_NCCL(ctx, api->Recv((char *)out->cols[c].nulls + roff[(size_t)peer] + r0, (size_t)(r1 - r0), ncclInt8, peer, cm, st));
                    }
                }
            }
            GSQL_NCCL(ctx, api->GroupEnd());
        }
        for (int k = 1; k < K; k++) {  // join the stripes back into the context stream
            cudaEvent_t done;
            GSQL_CUDA(ctx, cudaEventCreateWithFlags(&done, cudaEventDisableTiming));
            GSQL_CUDA(ctx, cudaEventRecord(done, ctx->xstreams[k - 1]));
            GSQL_CUDA(ctx, cudaStreamWaitEvent(ctx->stream, done, 0));
            GSQL_CUDA(ctx, cudaEventDestroy(done));
        }
        GSQL_CUDA(ctx, cudaEventDestroy(ready));
    }
    out->rows = total;
    return GSQL_OK;
}


// ================================================================================================ partition-and-push
// One-pass shuffle over peer-mapped memory (gsql_xchg_open_p2p / _push / _recv_view).  Per rank ONE device allocation
// holds a control block and the receive columns; CUDA IPC maps it into every peer.  A push:
//   1. k_xchg_hist per slab (keys only) + exclusive scan  -> rows per (slab, destination, block)
//   2. k_p2p_publish: every rank writes its counts[slab][dst] into every peer's control block, then all ranks meet in a
//      flag barrier (st.release.sys / ld.acquire.sys on the peer-mapped flags) -> each rank reads the whole
//      counts[src][slab][dst] matrix locally and derives, on the host, where every (src, slab) segment starts in every
//      receive buffer (gsql_xchg_plan_layout): slab-major, source-minor, so a slab is one contiguous batch.
//   3. per slab k_xchg_push_w (at most 4 columns, none nullable: a warp splits 256-row tiles by destination in its own
//      shared memory) or k_xchg_push (any other batch: a block splits 2048-row tiles, warp match.any ranks, one block
//      scan of the (destination, warp, row-slot) cells); either writes each destination's run of every column with
//      coalesced stores straight into that GPU's receive buffer over NVLink (self = local HBM); then k_p2p_barrier.
// No staging buffer, no NCCL kernel on the data path; the consumer of slab k (join probe, aggregation) runs on the
// context stream while slab k+1 is being pushed on the exchange's stream.
namespace {

constexpr int PUSH_THREADS = 512;
constexpr int PUSH_RPT = 4;
constexpr int PUSH_TILE = PUSH_THREADS * PUSH_RPT;
constexpr int PUSH_WARPS = PUSH_THREADS / 32;
constexpr int PUSH_CELLS = PUSH_WARPS * PUSH_RPT;  // (warp, row-slot) cells per destination
constexpr size_t CTRL_BYTES = 512 * 1024;

}  // namespace

struct P2PCtrl {                                   // first bytes of every rank's peer-mapped allocation
    unsigned long long flag[GSQL_MAX_RANKS];       // flag[src]: last barrier sequence number rank src arrived at
    int32_t err;                                   // local only: a barrier timed out
    int32_t pad[31];
    long long counts[2][GSQL_MAX_RANKS][GSQL_MAX_SLABS][GSQL_MAX_RANKS];  // [push parity][src][slab][dst], written by src
};
static_assert(sizeof(P2PCtrl) <= CTRL_BYTES, "control block must fit its region");

namespace {

struct PeerSet {
    P2PCtrl *ctrl[GSQL_MAX_RANKS];
    int32_t nranks, me;
};

__device__ __forceinline__ void st_release_sys(unsigned long long *p, unsigned long long v) {
    asm volatile("st.release.sys.global.u64 [%0], %1;" ::"l"(p), "l"(v) : "memory");
}
__device__ __forceinline__ unsigned long long ld_acquire_sys(const unsigned long long *p) {
    unsigned long long v;
    asm volatile("ld.acquire.sys.global.u64 %0, [%1];" : "=l"(v) : "l"(p) : "memory");
    return v;
}
__device__ __forceinline__ unsigned long long global_timer_ns() {
    unsigned long long t;
    asm volatile("mov.u64 %0, %globaltimer;" : "=l"(t));
    return t;
}

// All ranks meet: thread t tells rank t "I arrived at seq" and waits until rank t has told this rank the same.  Everything
// this rank wrote to peer memory before (earlier kernels of the stream, or this kernel before the __syncthreads) is
// visible to a peer that has passed its own barrier.  Bounded: a peer that never arrives sets err instead of hanging.
__device__ __forceinline__ void p2p_barrier(const PeerSet &S, unsigned long long seq) {
    __syncthreads();
    if ((int)threadIdx.x < S.nranks) {
        __threadfence_system();
        st_release_sys(&S.ctrl[threadIdx.x]->flag[S.me], seq);
        const unsigned long long t0 = global_timer_ns();
        while (ld_acquire_sys(&S.ctrl[S.me]->flag[threadIdx.x]) < seq) {
            __nanosleep(200);
            if (global_timer_ns() - t0 > 30000000000ULL) {  // 30 s
                S.ctrl[S.me]->err = 1;
                break;
            }
        }
    }
    __syncthreads();
}

struct SlabOffs {
    const int64_t *offs[GSQL_MAX_SLABS];  // [dst][block] exclusive scan of slab i (+ one total entry)
    int64_t fixed[GSQL_MAX_SLABS];        // >= 0: every destination receives this many rows of slab i (broadcast)
    int32_t nblocks[GSQL_MAX_SLABS];
    int32_t nslabs, parity;
};

__global__ void __launch_bounds__(256) k_p2p_publish(const __grid_constant__ PeerSet S, const __grid_constant__ SlabOffs O, unsigned long long seq) {
    const int R = S.nranks;
    for (int i = threadIdx.x; i < O.nslabs * R; i += blockDim.x) {
        const int slab = i / R, dst = i % R;
        const int64_t *o = O.offs[slab];
        const int nb = O.nblocks[slab];
        const long long cnt = O.fixed[slab] >= 0 ? (long long)O.fixed[slab] : (long long)(o[(int64_t)(dst + 1) * nb] - o[(int64_t)dst * nb]);
        for (int p = 0; p < R; p++) S.ctrl[p]->counts[O.parity][S.me][slab][dst] = cnt;
    }
    p2p_barrier(S, seq);
}

__global__ void __launch_bounds__(32) k_p2p_barrier(const __grid_constant__ PeerSet S, unsigned long long seq) { p2p_barrier(S, seq); }

struct PushParams {
    XParams X;                              // the slab: input columns, key channels, nparts = ranks, block geometry
    const int64_t *offs;                    // [dst][block] exclusive scan of this slab
    int64_t base_row[GSQL_MAX_RANKS];       // first row of this rank's (slab) segment in dst's receive buffer
    char *peer_base[GSQL_MAX_RANKS];        // dst's allocation, mapped here
    int64_t col_off[GSQL_MAX_COLS];         // byte offset of column c inside an allocation
    int64_t null_off[GSQL_MAX_COLS];        // byte offset of column c's NULL bytes, or -1
};

// Destination of row r.  FAST: one integer key column without a NULL buffer, hash mode — the shape of every join / group
// key exchange in the benchmarks; everything else goes through the generic row hash.
constexpr int XMODE_SLOT_RANGE = 100;  // internal: destination = mulhi(fmix64(key), nparts) (local_split_by_slot_range)

template <bool FAST>
__device__ __forceinline__ int push_dest(const XParams &P, int64_t r) {
    if (FAST) {
        const DCol &c = P.keys.c[0];
        if (P.mode == XMODE_SLOT_RANGE) {  // block-uniform
            const long long v = c.type == GSQL_T_INT32 ? (long long)ld_stream_4(reinterpret_cast<const int *>(c.data) + r)
                                                       : ld_stream_8(reinterpret_cast<const long long *>(c.data) + r);
            return (int)__umul64hi(gsql_fmix64((unsigned long long)v), (unsigned long long)P.nparts);
        }
        int32_t h;
        if (c.type == GSQL_T_INT32) {
            const int v = ld_stream_4(reinterpret_cast<const int *>(c.data) + r);
            h = P.keys.utype[0] == GSQL_T_INT32 ? v : gsql_hash_i64((int64_t)v);
        } else {
            h = gsql_hash_i64(ld_stream_8(reinterpret_cast<const long long *>(c.data) + r));
        }
        return gsql_partition_of(h, P.nparts, P.pow2 != 0);
    }
    return row_part(P, r);
}

static bool push_fast_key(const XParams &X) {
    return (X.mode == GSQL_XCHG_HASH || X.mode == XMODE_SLOT_RANGE) && X.keys.n == 1 && X.keys.c[0].nulls == nullptr && X.keys.c[0].type != GSQL_T_FP64 &&
           X.keys.utype[0] != GSQL_T_FP64 && !(X.keys.c[0].type == GSQL_T_INT64 && X.keys.utype[0] == GSQL_T_INT32);
}

// hist[dst * nblocks + b] = rows of block b's chunk routed to dst.  Same block geometry as k_xchg_push.  Four rows per
// thread are in flight; a warp adds one shared-memory count per distinct destination (match.any), not one per row.
template <bool FAST>
__global__ void __launch_bounds__(PUSH_THREADS) k_push_hist(const __grid_constant__ XParams P, int64_t *__restrict__ hist) {
    __shared__ unsigned int sh[GSQL_MAX_RANKS];
    const int tid = threadIdx.x, lane = tid & 31;
    if (tid < GSQL_MAX_RANKS) sh[tid] = 0;
    __syncthreads();
    const int64_t r0 = (int64_t)blockIdx.x * P.chunk;
    const int64_t r1 = r0 + P.chunk < P.rows ? r0 + P.chunk : P.rows;
    for (int64_t t0 = r0; t0 < r1; t0 += PUSH_TILE) {
        int d[PUSH_RPT];
#pragma unroll
        for (int k = 0; k < PUSH_RPT; k++) {
            const int64_t r = t0 + k * PUSH_THREADS + tid;
            d[k] = r < r1 ? push_dest<FAST>(P, r) : -1;
        }
#pragma unroll
        for (int k = 0; k < PUSH_RPT; k++) {
            const unsigned peers = __match_any_sync(0xffffffffu, d[k]);
            if (d[k] >= 0 && (peers & ((1u << lane) - 1u)) == 0) atomicAdd(&sh[d[k]], (unsigned)__popc(peers));
        }
    }
    __syncthreads();
    if (tid < P.nparts) hist[(int64_t)tid * P.nblocks + blockIdx.x] = sh[tid];
}

// Block-synchronous split for the batches k_xchg_push_w does not take (NULL masks, or more than 4 columns): a 2048-row
// tile is ranked by destination once, then its columns are staged and flushed one after another.
template <bool FAST>
__global__ void __launch_bounds__(PUSH_THREADS, 2) k_xchg_push(const __grid_constant__ PushParams P) {
    __shared__ __align__(16) unsigned long long stage[2][PUSH_TILE];  // one column of the tile in destination order (double-buffered)
    __shared__ unsigned char sdest[PUSH_TILE];                        // destination of each staged position
    __shared__ unsigned int cell[GSQL_MAX_RANKS * PUSH_CELLS];        // rows per (dst, warp, slot) -> exclusive starts
    __shared__ unsigned long long cur[GSQL_MAX_RANKS];                // next row of this block in dst's receive buffer
    __shared__ unsigned int dstart[GSQL_MAX_RANKS + 1];
    typedef cub::BlockScan<unsigned int, PUSH_THREADS> BlockScan;
    __shared__ typename BlockScan::TempStorage scan_tmp;
    const int R = P.X.nparts;
    const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
    const int nb = P.X.nblocks;
    if (tid < R) cur[tid] = (unsigned long long)(P.base_row[tid] + (P.offs[(int64_t)tid * nb + blockIdx.x] - P.offs[(int64_t)tid * nb]));
    const int64_t r0 = (int64_t)blockIdx.x * P.X.chunk;
    const int64_t r1 = r0 + P.X.chunk < P.X.rows ? r0 + P.X.chunk : P.X.rows;
    constexpr int IPT = GSQL_MAX_RANKS * PUSH_CELLS / PUSH_THREADS;  // cells per thread in the scan
    for (int64_t t0 = r0; t0 < r1; t0 += PUSH_TILE) {
        const int n_tile = (int)(r1 - t0 < PUSH_TILE ? r1 - t0 : PUSH_TILE);
        for (int i = tid; i < R * PUSH_CELLS; i += PUSH_THREADS) cell[i] = 0;
        // 1. destination of this thread's rows
        int d[PUSH_RPT];
        unsigned int rank[PUSH_RPT];
#pragma unroll
        for (int k = 0; k < PUSH_RPT; k++) {
            const int64_t r = t0 + k * PUSH_THREADS + tid;
            d[k] = r < r1 ? push_dest<FAST>(P.X, r) : -1;
        }
        __syncthreads();  // cells are zero; also orders the previous tile's last flush / cur update before this tile's writes
        // 2. rank among the warp's rows with the same destination; per (dst, warp, slot) counts
#pragma unroll
        for (int k = 0; k < PUSH_RPT; k++) {
            const unsigned peers = __match_any_sync(0xffffffffu, d[k]);
            rank[k] = __popc(peers & ((1u << lane) - 1u));
            if (d[k] >= 0 && rank[k] == 0) cell[d[k] * PUSH_CELLS + warp * PUSH_RPT + k] = __popc(peers);
        }
        __syncthreads();
        {  // exclusive scan of the cells in (dst, warp, slot) order: a destination's rows become one run of the tile
            unsigned int v[IPT];
#pragma unroll
            for (int i = 0; i < IPT; i++) {
                const int c = tid * IPT + i;
                v[i] = c < R * PUSH_CELLS ? cell[c] : 0;
            }
            BlockScan(scan_tmp).ExclusiveSum(v, v);
#pragma unroll
            for (int i = 0; i < IPT; i++) {
                const int c = tid * IPT + i;
                if (c < R * PUSH_CELLS) {
                    cell[c] = v[i];
                    if (c % PUSH_CELLS == 0) dstart[c / PUSH_CELLS] = v[i];
                }
            }
            if (tid == 0) dstart[R] = (unsigned int)n_tile;
        }
        __syncthreads();
        unsigned int pos[PUSH_RPT];
#pragma unroll
        for (int k = 0; k < PUSH_RPT; k++) {
            pos[k] = 0;
            if (d[k] >= 0) {
                pos[k] = cell[d[k] * PUSH_CELLS + warp * PUSH_RPT + k] + rank[k];
                sdest[pos[k]] = (unsigned char)d[k];
            }
        }
        // 3. column after column: stage in destination order, then consecutive threads store consecutive elements of a
        //    destination's run into that GPU's receive buffer
        int phase = 0;
        auto flush = [&](int c, bool is32, const unsigned long long *st, bool nulls) {
#pragma unroll
            for (int k = 0; k < PUSH_RPT; k++) {
                const int i = k * PUSH_THREADS + tid;
                if (i < n_tile) {
                    const int dd = sdest[i];
                    const unsigned long long row = cur[dd] + (unsigned)(i - (int)dstart[dd]);
                    if (nulls) reinterpret_cast<uint8_t *>(P.peer_base[dd] + P.null_off[c])[row] = (uint8_t)st[i];
                    else if (is32) reinterpret_cast<int *>(P.peer_base[dd] + P.col_off[c])[row] = (int)(unsigned)st[i];
                    else reinterpret_cast<long long *>(P.peer_base[dd] + P.col_off[c])[row] = (long long)st[i];
                }
            }
        };
#pragma unroll 1
        for (int c = 0; c < P.X.in.n; c++) {
            const DCol &col = P.X.in.c[c];
            const bool is32 = col.type == GSQL_T_INT32;
            unsigned long long v[PUSH_RPT];
#pragma unroll
            for (int k = 0; k < PUSH_RPT; k++) {
                const int64_t r = t0 + k * PUSH_THREADS + tid;
                v[k] = 0;
                if (d[k] >= 0) v[k] = is32 ? (unsigned long long)(unsigned)ld_stream_4(reinterpret_cast<const int *>(col.data) + r)
                                           : (unsigned long long)ld_stream_8(reinterpret_cast<const long long *>(col.data) + r);
            }
            unsigned long long *st = stage[phase];
#pragma unroll
            for (int k = 0; k < PUSH_RPT; k++)
                if (d[k] >= 0) st[pos[k]] = v[k];
            __syncthreads();
            flush(c, is32, st, false);
            phase ^= 1;
            if (P.null_off[c] >= 0) {  // NULL bytes travel the same way
                unsigned long long *sn = stage[phase];
#pragma unroll
                for (int k = 0; k < PUSH_RPT; k++) {
                    const int64_t r = t0 + k * PUSH_THREADS + tid;
                    if (d[k] >= 0) sn[pos[k]] = col.nulls ? (unsigned long long)col.nulls[r] : 0ULL;
                }
                __syncthreads();
                flush(c, false, sn, true);
                phase ^= 1;
            }
        }
        __syncthreads();
        if (tid < R) cur[tid] += dstart[tid + 1] - dstart[tid];
    }
}

// Warp-synchronous split for NC <= 4 columns without NULL masks (the join / group-by exchanges of the benchmarks): no
// block barrier in the row loop.  A warp takes 256 rows (8 per lane, all loads in flight), splits them by
// destination inside its PRIVATE 6 KB of shared memory (match.any ranks per row slot, running per-destination offsets in
// warp-private counters), reserves its rows in every destination's run of the block with one shared-memory atomic per
// destination, and writes each destination's ~256/R rows of every column as one contiguous run (>= 128 bytes for R <= 8)
// into that GPU's receive buffer.  Warps never wait for each other, so the load latency of one warp hides behind the
// split and the stores of the others; k_xchg_push above needs four block barriers per 2048-row tile plus one per
// column and NULL mask.
constexpr int PW_RPL = 8;                 // rows per lane per warp tile
constexpr int PW_TILE = 32 * PW_RPL;      // 256 rows per warp tile
constexpr int PW_WARPS = 4;               // 128 threads per block: <= 32 KB of staging, five blocks per SM

template <bool FAST, int NC>
__global__ void __launch_bounds__(PW_WARPS * 32, 8) k_xchg_push_w(const __grid_constant__ PushParams P) {
    __shared__ __align__(16) unsigned long long wstage[PW_WARPS][NC][PW_TILE];  // a warp's tile, column-major, in destination order
    __shared__ unsigned int wcnt[PW_WARPS][GSQL_MAX_RANKS];
    __shared__ unsigned int wgo[PW_WARPS][GSQL_MAX_RANKS + 1];
    __shared__ unsigned long long wg[PW_WARPS][GSQL_MAX_RANKS];
    __shared__ unsigned long long cur[GSQL_MAX_RANKS];
    const int R = P.X.nparts;
    const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
    const int nb = P.X.nblocks;
    if (tid < R) cur[tid] = (unsigned long long)(P.base_row[tid] + (P.offs[(int64_t)tid * nb + blockIdx.x] - P.offs[(int64_t)tid * nb]));
    __syncthreads();
    const int64_t r0 = (int64_t)blockIdx.x * P.X.chunk;
    const int64_t r1 = r0 + P.X.chunk < P.X.rows ? r0 + P.X.chunk : P.X.rows;
    for (int64_t t0 = r0 + (int64_t)warp * PW_TILE; t0 < r1; t0 += (int64_t)PW_WARPS * PW_TILE) {
        const int n_tile = (int)(r1 - t0 < PW_TILE ? r1 - t0 : PW_TILE);
        // ---- 1. destinations (the key loads of all eight rows are in flight together)
        int d[PW_RPL];
#pragma unroll
        for (int k = 0; k < PW_RPL; k++) {
            const int64_t r = t0 + k * 32 + lane;
            d[k] = r < r1 ? push_dest<FAST>(P.X, r) : -1;
        }
        if (lane < GSQL_MAX_RANKS) wcnt[warp][lane] = 0;
        __syncwarp();
        // ---- 2. offset of every row inside its destination's part of the warp tile
        unsigned int off[PW_RPL];
#pragma unroll
        for (int k = 0; k < PW_RPL; k++) {
            const unsigned peers = __match_any_sync(0xffffffffu, d[k]);
            const int leader = __ffs(peers) - 1;
            unsigned int before = 0;
            if (d[k] >= 0 && lane == leader) {
                before = wcnt[warp][d[k]];
                wcnt[warp][d[k]] = before + __popc(peers);
            }
            before = __shfl_sync(0xffffffffu, before, leader);
            off[k] = before + __popc(peers & ((1u << lane) - 1u));
            __syncwarp();
        }
        // exclusive scan of the per-destination counts; one reservation per destination in the block's runs
        {
            unsigned int c = lane < R ? wcnt[warp][lane] : 0;
            unsigned int incl = c;
#pragma unroll
            for (int s2 = 1; s2 < GSQL_MAX_RANKS; s2 <<= 1) {
                const unsigned int t = __shfl_up_sync(0xffffffffu, incl, s2);
                if (lane >= s2) incl += t;
            }
            if (lane < R) {
                wgo[warp][lane] = incl - c;
                wg[warp][lane] = c ? atomicAdd(&cur[lane], (unsigned long long)c) : 0ULL;
            }
            if (lane == 0) wgo[warp][R] = (unsigned int)n_tile;
        }
        __syncwarp();
#pragma unroll
        for (int k = 0; k < PW_RPL; k++) off[k] += d[k] >= 0 ? wgo[warp][d[k]] : 0u;  // position in the staged tile
        // ---- 3. column after column: eight loads in flight per lane, staged in destination order
#pragma unroll
        for (int c = 0; c < NC; c++) {
            const DCol &col = P.X.in.c[c];
            const bool is32 = col.type == GSQL_T_INT32;
            unsigned long long v[PW_RPL];
#pragma unroll
            for (int k = 0; k < PW_RPL; k++) {
                const int64_t r = t0 + k * 32 + lane;
                v[k] = 0;
                if (d[k] >= 0) v[k] = is32 ? (unsigned long long)(unsigned)ld_stream_4(reinterpret_cast<const int *>(col.data) + r)
                                           : (unsigned long long)ld_stream_8(reinterpret_cast<const long long *>(col.data) + r);
            }
#pragma unroll
            for (int k = 0; k < PW_RPL; k++)
                if (d[k] >= 0) wstage[warp][c][off[k]] = v[k];
        }
        __syncwarp();
        // ---- 4. flush: staged position i belongs to the destination whose range [wgo[dd], wgo[dd+1]) holds it; its row in
        //         that GPU's receive buffer is computed once and used for every column
#pragma unroll
        for (int k = 0; k < PW_RPL; k++) {
            const int i = k * 32 + lane;
            if (i < n_tile) {
                int dd = 0;
#pragma unroll
                for (int q = 1; q < GSQL_MAX_RANKS; q++)
                    if (q < R && (unsigned)i >= wgo[warp][q]) dd = q;
                const unsigned long long row = wg[warp][dd] + (unsigned)(i - (int)wgo[warp][dd]);
                char *base = P.peer_base[dd];
#pragma unroll
                for (int c = 0; c < NC; c++) {
                    if (P.X.in.c[c].type == GSQL_T_INT32) reinterpret_cast<int *>(base + P.col_off[c])[row] = (int)(unsigned)wstage[warp][c][i];
                    else reinterpret_cast<long long *>(base + P.col_off[c])[row] = (long long)wstage[warp][c][i];
                }
            }
        }
        __syncwarp();
    }
}

// distribution=broadcast: the slab's rows are read once and stored into EVERY rank's receive buffer (this rank's segment
// of it).  Column after column, grid-stride, one element per thread: every store instruction writes a contiguous run.
__global__ void __launch_bounds__(256) k_xchg_bcast(const __grid_constant__ PushParams P) {
    const int R = P.X.nparts;
    const int64_t stride = (int64_t)gridDim.x * blockDim.x, first = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
    for (int c = 0; c < P.X.in.n; c++) {
        const DCol &col = P.X.in.c[c];
        if (col.type == GSQL_T_INT32) {
            for (int64_t i = first; i < P.X.rows; i += stride) {
                const int v = ld_stream_4(reinterpret_cast<const int *>(col.data) + i);
                for (int d = 0; d < R; d++) reinterpret_cast<int *>(P.peer_base[d] + P.col_off[c])[P.base_row[d] + i] = v;
            }
        } else {
            for (int64_t i = first; i < P.X.rows; i += stride) {
                const long long v = ld_stream_8(reinterpret_cast<const long long *>(col.data) + i);
                for (int d = 0; d < R; d++) reinterpret_cast<long long *>(P.peer_base[d] + P.col_off[c])[P.base_row[d] + i] = v;
            }
        }
        if (P.null_off[c] >= 0)
            for (int64_t i = first; i < P.X.rows; i += stride) {
                const uint8_t v = col.nulls ? col.nulls[i] : 0;
                for (int d = 0; d < R; d++) reinterpret_cast<uint8_t *>(P.peer_base[d] + P.null_off[c])[P.base_row[d] + i] = v;
            }
    }
}

}  // namespace

extern "C" int64_t gsql_xchg_plan_layout(int32_t nranks, int32_t nslabs, int32_t me, const int64_t *matrix, int64_t *send_base,
                                         int64_t *recv_base, int64_t *slab_rows) {
    if (nranks < 1 || nslabs < 1 || me < 0 || me >= nranks || !matrix) return -1;
    auto m_at = [&](int src, int slab, int dst) -> int64_t { return matrix[((size_t)src * nslabs + slab) * nranks + dst]; };
    int64_t worst = 0;
    for (int dst = 0; dst < nranks; dst++) {
        int64_t row = 0;  // dst's buffer: slab after slab; inside a slab, source after source
        for (int slab = 0; slab < nslabs; slab++) {
            const int64_t slab_first = row;
            for (int src = 0; src < nranks; src++) {
                if (src == me && send_base) send_base[(size_t)slab * nranks + dst] = row;
                if (dst == me && recv_base) recv_base[(size_t)slab * nranks + src] = row;
                row += m_at(src, slab, dst);
            }
            if (dst == me && slab_rows) slab_rows[slab] = row - slab_first;
        }
        if (row > worst) worst = row;
    }
    return worst;
}

static void p2p_close(gsql_xchg *x) {
    if (!x->p2p) return;
    gsql_ctx *ctx = x->ctx;
    if (x->pstream) cudaStreamSynchronize(x->pstream);
    cudaStreamSynchronize(ctx->stream);
    for (int r = 0; r < ctx->nranks; r++)
        if (r != ctx->rank && x->peer_base[r]) cudaIpcCloseMemHandle(x->peer_base[r]);
    if (x->base) cudaFree(x->base);
    if (x->in_ev) cudaEventDestroy(x->in_ev);
    for (int i = 0; i < GSQL_MAX_SLABS; i++)
        if (x->slab_ev[i]) cudaEventDestroy(x->slab_ev[i]);
    if (x->pstream) cudaStreamDestroy(x->pstream);
    if (x->host_matrix) cudaFreeHost(x->host_matrix);
    if (x->host_err) cudaFreeHost(x->host_err);
    x->p2p = false;
    x->base = nullptr;
}

extern "C" gsql_status gsql_xchg_open_p2p(gsql_xchg *x, int64_t recv_capacity_rows, uint32_t nullable_cols) {
    if (!x || recv_capacity_rows < 1) return GSQL_E_INVALID;
    gsql_ctx *ctx = x->ctx;
    if (ctx->sticky) return GSQL_E_CUDA;
    const gsql_xchg_spec &s = x->spec;
    const int R = ctx->nranks;
    if (x->p2p) return gsql_set_error(ctx, GSQL_E_STATE, "exchange is already open");
    if (R > GSQL_MAX_RANKS) return gsql_set_error(ctx, GSQL_E_UNSUPPORTED, "at most %d ranks", GSQL_MAX_RANKS);
    if (s.nparts != R) return gsql_set_error(ctx, GSQL_E_INVALID, "exchange has %d partitions but the communicator has %d ranks", s.nparts, R);
    NcclApi *api = nccl_api();
    if (R > 1 && (!ctx->nccl_comm || !api->ok)) return gsql_set_error(ctx, GSQL_E_STATE, "gsql_comm_init has not been called");
    GSQL_CUDA(ctx, cudaSetDevice(ctx->device));
    // ---- layout of the allocation: control block | column 0 | column 1 | ... | NULL bytes of the nullable columns
    size_t off = CTRL_BYTES;
    for (int c = 0; c < s.n_cols; c++) {
        x->col_off[c] = (int64_t)off;
        off += ((size_t)recv_capacity_rows * gsql_type_width(s.types[c]) + 255) & ~(size_t)255;
    }
    for (int c = 0; c < s.n_cols; c++) {
        x->null_off[c] = -1;
        if (nullable_cols & (1u << c)) {
            x->null_off[c] = (int64_t)off;
            off += ((size_t)recv_capacity_rows + 255) & ~(size_t)255;
        }
    }
    x->alloc_bytes = off;
    x->cap = recv_capacity_rows;
    {
        cudaError_t e = cudaMalloc((void **)&x->base, off);  // not from the stream-ordered pool: IPC needs a plain allocation
        if (e != cudaSuccess) {
            cudaGetLastError();
            x->base = nullptr;
            return gsql_set_error(ctx, GSQL_E_OOM, "cudaMalloc(%zu bytes) for the receive buffer: %s", off, cudaGetErrorString(e));
        }
    }
    x->p2p = true;  // from here on p2p_close releases everything
    GSQL_CUDA(ctx, cudaMemset(x->base, 0, CTRL_BYTES));
    GSQL_CUDA(ctx, cudaDeviceSynchronize());
    int lo = 0, hi = 0;
    cudaDeviceGetStreamPriorityRange(&lo, &hi);
    GSQL_CUDA(ctx, cudaStreamCreateWithPriority(&x->pstream, cudaStreamNonBlocking, hi));
    GSQL_CUDA(ctx, cudaEventCreateWithFlags(&x->in_ev, cudaEventDisableTiming));
    for (int i = 0; i < GSQL_MAX_SLABS; i++) GSQL_CUDA(ctx, cudaEventCreateWithFlags(&x->slab_ev[i], cudaEventDisableTiming));
    GSQL_CUDA(ctx, cudaHostAlloc((void **)&x->host_matrix, sizeof(long long) * GSQL_MAX_RANKS * GSQL_MAX_SLABS * GSQL_MAX_RANKS, cudaHostAllocDefault));
    GSQL_CUDA(ctx, cudaHostAlloc((void **)&x->host_err, 64, cudaHostAllocDefault));
    for (int r = 0; r < GSQL_MAX_RANKS; r++) x->peer_base[r] = nullptr;
    x->peer_base[ctx->rank] = x->base;
    if (R > 1) {  // exchange the IPC handles (NCCL is plumbing here: 64 bytes per rank, once)
        cudaIpcMemHandle_t mine;
        GSQL_CUDA(ctx, cudaIpcGetMemHandle(&mine, x->base));
        DevBuf d_mine, d_all;
        GSQL_TRY(d_mine.alloc(ctx, sizeof(mine)));
        GSQL_TRY(d_all.alloc(ctx, sizeof(mine) * (size_t)R));
        GSQL_CUDA(ctx, cudaMemcpyAsync(d_mine.p, &mine, sizeof(mine), cudaMemcpyHostToDevice, ctx->stream));
        GSQL_NCCL(ctx, api->AllGather(d_mine.p, d_all.p, sizeof(mine), ncclInt8, (ncclComm_t)ctx->nccl_comm, ctx->stream));
        std::vector<cudaIpcMemHandle_t> all((size_t)R);
        GSQL_CUDA(ctx, cudaMemcpyAsync(all.data(), d_all.p, sizeof(mine) * (size_t)R, cudaMemcpyDeviceToHost, ctx->stream));
        GSQL_CUDA(ctx, cudaStreamSynchronize(ctx->stream));  // every rank zeroed its control block before contributing
        for (int r = 0; r < R; r++) {
            if (r == ctx->rank) continue;
            void *p = nullptr;
            cudaError_t e = cudaIpcOpenMemHandle(&p, all[(size_t)r], cudaIpcMemLazyEnablePeerAccess);
            if (e != cudaSuccess) {
                cudaGetLastError();
                return gsql_set_error(ctx, GSQL_E_CUDA, "cudaIpcOpenMemHandle(rank %d): %s — peer access over NVLink is required", r, cudaGetErrorString(e));
            }
            x->peer_base[r] = (char *)p;
        }
    }
    return GSQL_OK;
}

static void fill_peers(gsql_xchg *x, PeerSet *S) {
    memset(S, 0, sizeof(*S));
    S->nranks = x->ctx->nranks;
    S->me = x->ctx->rank;
    for (int r = 0; r < S->nranks; r++) S->ctrl[r] = reinterpret_cast<P2PCtrl *>(x->peer_base[r]);
}

// nc = 1..4: the batch's columns, none of them nullable -> k_xchg_push_w; nc = 0: any other batch -> k_xchg_push
template <bool FAST>
static void launch_push(const PushParams &PP, int nc, int nblocks, cudaStream_t ps) {
    switch (nc) {
    case 1: k_xchg_push_w<FAST, 1><<<nblocks, PW_WARPS * 32, 0, ps>>>(PP); break;
    case 2: k_xchg_push_w<FAST, 2><<<nblocks, PW_WARPS * 32, 0, ps>>>(PP); break;
    case 3: k_xchg_push_w<FAST, 3><<<nblocks, PW_WARPS * 32, 0, ps>>>(PP); break;
    case 4: k_xchg_push_w<FAST, 4><<<nblocks, PW_WARPS * 32, 0, ps>>>(PP); break;
    default: k_xchg_push<FAST><<<nblocks, PUSH_THREADS, 0, ps>>>(PP); break;
    }
}

static int push_blocks(gsql_ctx *ctx, int64_t rows) {
    int per_sm = 8;
    if (const char *e = getenv("GSQL_XCHG_PUSH_CTAS_PER_SM")) per_sm = atoi(e);
    if (per_sm < 1) per_sm = 1;
    int64_t nb = (int64_t)ctx->sm_count * per_sm;
    if (const char *e = getenv("GSQL_XCHG_PUSH_CTAS")) nb = atoll(e);  // fewer CTAs leave more of the GPU to the overlapped consumer
    int64_t tiles = div_up(rows > 0 ? rows : 1, PUSH_TILE);
    if (nb > tiles) nb = tiles;
    if (nb < 1) nb = 1;
    return (int)nb;
}

extern "C" gsql_status gsql_xchg_push(gsql_xchg *x, const gsql_batch *in, int32_t nslabs, int64_t *slab_rows, int64_t *total_rows) {
    if (!x || !in) return GSQL_E_INVALID;
    gsql_ctx *ctx = x->ctx;
    if (ctx->sticky) return GSQL_E_CUDA;
    if (!x->p2p) return gsql_set_error(ctx, GSQL_E_STATE, "gsql_xchg_open_p2p has not been called");
    const gsql_xchg_spec &s = x->spec;
    GSQL_TRY(validate_batch(ctx, in, s.n_cols, s.types));
    if (in->mem != GSQL_MEM_DEVICE) return gsql_set_error(ctx, GSQL_E_INVALID, "push works on device-resident batches");
    if (nslabs < 1 || nslabs > GSQL_MAX_SLABS) return gsql_set_error(ctx, GSQL_E_INVALID, "1..%d slabs", GSQL_MAX_SLABS);
    for (int c = 0; c < s.n_cols; c++)
        if (in->cols[c].nulls && x->null_off[c] < 0) return gsql_set_error(ctx, GSQL_E_INVALID, "column %d carries NULLs but the exchange was opened without a mask for it", c);
    GSQL_CUDA(ctx, cudaSetDevice(ctx->device));
    const int R = ctx->nranks, me = ctx->rank;
    const int64_t n = in->rows;
    StagedBatch sb;
    GSQL_TRY(stage_batch(ctx, in, &sb));
    // rows per slab: a multiple of the tile, the last slabs may be short or empty
    const int64_t SR = div_up(div_up(n > 0 ? n : 1, nslabs), PUSH_TILE) * PUSH_TILE;
    std::vector<XParams> XP((size_t)nslabs);
    std::vector<int64_t> rows_of((size_t)nslabs, 0);
    size_t tmp_bytes = 0;
    bool regrow = false;
    for (int i = 0; i < nslabs; i++) {
        const int64_t lo = (int64_t)i * SR;
        rows_of[(size_t)i] = lo < n ? (n - lo < SR ? n - lo : SR) : 0;
        fill_xparams(x, sb, lo < n ? lo : 0, rows_of[(size_t)i], &XP[(size_t)i]);
        XParams &X = XP[(size_t)i];
        int nb = push_blocks(ctx, X.rows);
        X.chunk = div_up(div_up(X.rows > 0 ? X.rows : 1, nb), PUSH_TILE) * PUSH_TILE;
        nb = (int)div_up(X.rows, X.chunk);
        X.nblocks = nb < 1 ? 1 : nb;
        const int64_t nh = (int64_t)R * X.nblocks;
        if (x->hist[i].bytes < (size_t)(nh + 1) * 8 || x->offs[i].bytes < (size_t)(nh + 1) * 8) regrow = true;
        size_t tb = 0;
        GSQL_CUDA(ctx, cub::DeviceScan::ExclusiveSum(nullptr, tb, (int64_t *)nullptr, (int64_t *)nullptr, nh + 1, x->pstream));
        if (tb > tmp_bytes) tmp_bytes = tb;
    }
    if (regrow || x->scan_tmp.bytes < tmp_bytes) {  // the scratch lives in the handle; it only grows, and never under a push in flight
        GSQL_CUDA(ctx, cudaStreamSynchronize(x->pstream));
        for (int i = 0; i < nslabs; i++) {
            const int64_t nh = (int64_t)R * XP[(size_t)i].nblocks;
            GSQL_TRY(x->hist[i].grow(ctx, (size_t)(nh + 1) * 8, 0));
            GSQL_TRY(x->offs[i].grow(ctx, (size_t)(nh + 1) * 8, 0));
        }
        GSQL_TRY(x->scan_tmp.grow(ctx, tmp_bytes ? tmp_bytes : 16, 0));
    }
    // the exchange stream starts after everything the caller enqueued on the context stream: the input exists, and
    // the consumers of the previous push's rows are done with the receive buffer (and so, after the publish barrier
    // below, are the consumers on every other rank: nobody overwrites rows that are still being read)
    GSQL_CUDA(ctx, cudaEventRecord(x->in_ev, ctx->stream));
    GSQL_CUDA(ctx, cudaStreamWaitEvent(x->pstream, x->in_ev, 0));
    cudaStream_t ps = x->pstream;
    // ---- 1. histograms + scans of every slab
    SlabOffs SO;
    memset(&SO, 0, sizeof(SO));
    SO.nslabs = nslabs;
    SO.parity = (int32_t)(x->pushes & 1);
    for (int i = 0; i < nslabs; i++) {
        XParams &X = XP[(size_t)i];
        const int64_t nh = (int64_t)R * X.nblocks;
        SO.offs[i] = x->offs[i].as<int64_t>();
        SO.nblocks[i] = X.nblocks;
        SO.fixed[i] = -1;
        if (s.mode == GSQL_XCHG_BROADCAST) {  // nothing to count: every destination receives the whole slab
            SO.fixed[i] = X.rows;
            continue;
        }
        GSQL_CUDA(ctx, cudaMemsetAsync(x->hist[i].p, 0, (size_t)(nh + 1) * 8, ps));
        if (X.rows > 0) {
            KernelScope ks(ctx, "xchg_push_hist", ps);
            if (push_fast_key(X)) k_push_hist<true><<<X.nblocks, PUSH_THREADS, 0, ps>>>(X, x->hist[i].as<int64_t>());
            else k_push_hist<false><<<X.nblocks, PUSH_THREADS, 0, ps>>>(X, x->hist[i].as<int64_t>());
        }
        size_t tb = x->scan_tmp.bytes;
        GSQL_CUDA(ctx, cub::DeviceScan::ExclusiveSum(x->scan_tmp.p, tb, x->hist[i].as<int64_t>(), x->offs[i].as<int64_t>(), nh + 1, ps));
    }
    GSQL_CUDA(ctx, cudaGetLastError());
    // ---- 2. publish the counts to every peer, meet, read the whole matrix
    PeerSet S;
    fill_peers(x, &S);
    ctx->launches++;
    k_p2p_publish<<<1, 256, 0, ps>>>(S, SO, ++x->seq);
    GSQL_CUDA(ctx, cudaGetLastError());
    P2PCtrl *my = reinterpret_cast<P2PCtrl *>(x->base);
    GSQL_CUDA(ctx, cudaMemcpyAsync(x->host_matrix, &my->counts[SO.parity][0][0][0], sizeof(long long) * GSQL_MAX_RANKS * GSQL_MAX_SLABS * GSQL_MAX_RANKS,
                                   cudaMemcpyDeviceToHost, ps));
    GSQL_CUDA(ctx, cudaMemcpyAsync(x->host_err, &my->err, 4, cudaMemcpyDeviceToHost, ps));
    GSQL_CUDA(ctx, cudaStreamSynchronize(ps));
    x->pushes++;
    if (*x->host_err) {
        ctx->sticky = true;
        return gsql_set_error(ctx, GSQL_E_NCCL, "peer barrier timed out: a rank did not join the push");
    }
    std::vector<int64_t> M((size_t)R * nslabs * R), send_base((size_t)nslabs * R), recv_base((size_t)nslabs * R);
    for (int src = 0; src < R; src++)
        for (int i = 0; i < nslabs; i++)
            for (int dst = 0; dst < R; dst++)
                M[((size_t)src * nslabs + i) * R + dst] = x->host_matrix[((size_t)src * GSQL_MAX_SLABS + i) * GSQL_MAX_RANKS + dst];
    const int64_t worst = gsql_xchg_plan_layout(R, nslabs, me, M.data(), send_base.data(), recv_base.data(), x->slab_rows);
    int64_t mine = 0;
    for (int i = 0; i < nslabs; i++) {
        x->slab_base[i] = mine;
        mine += x->slab_rows[i];
        if (slab_rows) slab_rows[i] = x->slab_rows[i];
    }
    x->last_slabs = nslabs;
    if (worst > x->cap) {  // the same verdict on every rank (same matrix, same capacity): nobody sends
        x->last_slabs = 0;
        if (total_rows) *total_rows = worst;
        return gsql_set_error(ctx, GSQL_E_CAPACITY, "push needs %lld receive rows on some rank, capacity %lld", (long long)worst, (long long)x->cap);
    }
    if (total_rows) *total_rows = mine;
    // ---- 3. slab after slab: split-and-push kernel, then all ranks meet; the slab's event releases its consumer
    for (int i = 0; i < nslabs; i++) {
        XParams &X = XP[(size_t)i];
        if (X.rows > 0) {
            PushParams PP;
            memset(&PP, 0, sizeof(PP));
            PP.X = X;
            PP.offs = x->offs[i].as<int64_t>();
            for (int d = 0; d < R; d++) {
                PP.base_row[d] = send_base[(size_t)i * R + d];
                PP.peer_base[d] = x->peer_base[d];
            }
            for (int c = 0; c < s.n_cols; c++) {
                PP.col_off[c] = x->col_off[c];
                PP.null_off[c] = x->null_off[c];
            }
            {
                KernelScope ks(ctx, s.mode == GSQL_XCHG_BROADCAST ? "xchg_bcast" : "xchg_push", ps);
                if (s.mode == GSQL_XCHG_BROADCAST) {
                    int64_t g = div_up(X.rows, 256);
                    if (g > (int64_t)ctx->sm_count * 4) g = (int64_t)ctx->sm_count * 4;
                    k_xchg_bcast<<<(int)g, 256, 0, ps>>>(PP);
                } else {
                    bool plain = s.n_cols <= 4;  // warp-synchronous kernel: few columns, none of them nullable
                    for (int c = 0; c < s.n_cols; c++) plain = plain && x->null_off[c] < 0;
                    const int nc = plain ? s.n_cols : 0;
                    if (push_fast_key(X)) launch_push<true>(PP, nc, X.nblocks, ps);
                    else launch_push<false>(PP, nc, X.nblocks, ps);
                }
            }
            GSQL_CUDA(ctx, cudaGetLastError());
        }
        ctx->launches++;
        k_p2p_barrier<<<1, 32, 0, ps>>>(S, ++x->seq);
        GSQL_CUDA(ctx, cudaGetLastError());
        GSQL_CUDA(ctx, cudaEventRecord(x->slab_ev[i], ps));
    }
    return GSQL_OK;
}

extern "C" gsql_status gsql_xchg_recv_view(gsql_xchg *x, int32_t slab, gsql_batch *view) {
    if (!x || !view || !view->cols) return GSQL_E_INVALID;
    gsql_ctx *ctx = x->ctx;
    if (!x->p2p || x->last_slabs < 1) return gsql_set_error(ctx, GSQL_E_STATE, "no push to receive from");
    if (slab < -1 || slab >= x->last_slabs) return gsql_set_error(ctx, GSQL_E_INVALID, "slab %d of %d", slab, x->last_slabs);
    const gsql_xchg_spec &s = x->spec;
    GSQL_CUDA(ctx, cudaSetDevice(ctx->device));
    const int last = slab < 0 ? x->last_slabs - 1 : slab;
    GSQL_CUDA(ctx, cudaStreamWaitEvent(ctx->stream, x->slab_ev[last], 0));
    int64_t first = 0, rows = 0;
    if (slab < 0) {
        for (int i = 0; i < x->last_slabs; i++) rows += x->slab_rows[i];
    } else {
        first = x->slab_base[slab];
        rows = x->slab_rows[slab];
    }
    view->rows = rows;
    view->ncols = s.n_cols;
    view->mem = GSQL_MEM_DEVICE;
    for (int c = 0; c < s.n_cols; c++) {
        view->cols[c].type = s.types[c];
        view->cols[c].reserved = 0;
        view->cols[c].data = x->base + x->col_off[c] + (size_t)first * gsql_type_width(s.types[c]);
        view->cols[c].nulls = x->null_off[c] >= 0 ? reinterpret_cast<uint8_t *>(x->base + x->null_off[c] + first) : nullptr;
    }
    return GSQL_OK;
}

extern "C" gsql_status gsql_xchg_push_wait(gsql_xchg *x) {
    if (!x) return GSQL_E_INVALID;
    gsql_ctx *ctx = x->ctx;
    if (!x->p2p) return gsql_set_error(ctx, GSQL_E_STATE, "gsql_xchg_open_p2p has not been called");
    GSQL_CUDA(ctx, cudaStreamSynchronize(x->pstream));
    P2PCtrl *my = reinterpret_cast<P2PCtrl *>(x->base);
    int32_t err = 0;
    GSQL_CUDA(ctx, cudaMemcpy(&err, &my->err, 4, cudaMemcpyDeviceToHost));
    if (err) {
        ctx->sticky = true;
        return gsql_set_error(ctx, GSQL_E_NCCL, "peer barrier timed out: a rank did not finish the push");
    }
    return GSQL_OK;
}


// ------------------------------------------------------------------------------------------------ local split (agg pre-pass)
gsql_status local_split_by_slot_range(gsql_ctx *ctx, const DColSet &in, int key_col, int64_t rows, int nparts, void *const *out_data) {
    if (nparts < 1 || nparts > GSQL_MAX_RANKS || in.n < 1 || in.n > 4 || rows < 1) return gsql_set_error(ctx, GSQL_E_INVALID, "local split: unsupported shape");
    XParams X;
    memset(&X, 0, sizeof(X));
    X.in = in;
    X.keys.n = 1;
    X.keys.c[0] = in.c[key_col];
    X.keys.utype[0] = in.c[key_col].type;
    X.nparts = nparts;
    X.mode = XMODE_SLOT_RANGE;
    X.rows = rows;
    int nb = push_blocks(ctx, rows);
    X.chunk = div_up(div_up(rows, nb), PUSH_TILE) * PUSH_TILE;
    nb = (int)div_up(rows, X.chunk);
    X.nblocks = nb < 1 ? 1 : nb;
    const int64_t nh = (int64_t)nparts * X.nblocks;
    DevBuf hist, offs, tmp;
    GSQL_TRY(hist.alloc(ctx, (size_t)(nh + 1) * 8));
    GSQL_TRY(offs.alloc(ctx, (size_t)(nh + 1) * 8));
    GSQL_CUDA(ctx, cudaMemsetAsync(hist.p, 0, (size_t)(nh + 1) * 8, ctx->stream));
    {
        KernelScope ks(ctx, "agg_part_hist");
        k_push_hist<true><<<X.nblocks, PUSH_THREADS, 0, ctx->stream>>>(X, hist.as<int64_t>());
    }
    GSQL_CUDA(ctx, cudaGetLastError());
    size_t tb = 0;
    GSQL_CUDA(ctx, cub::DeviceScan::ExclusiveSum(nullptr, tb, hist.as<int64_t>(), offs.as<int64_t>(), nh + 1, ctx->stream));
    GSQL_TRY(tmp.alloc(ctx, tb));
    GSQL_CUDA(ctx, cub::DeviceScan::ExclusiveSum(tmp.p, tb, hist.as<int64_t>(), offs.as<int64_t>(), nh + 1, ctx->stream));
    PushParams PP;
    memset(&PP, 0, sizeof(PP));
    PP.X = X;
    PP.offs = offs.as<int64_t>();
    // destination d's run of column c starts at out_data[c] + (rows of the destinations before d): the exclusive scan is
    // destination-major, so offs[d * nblocks] is exactly that — the kernel adds (offs[d*nb + block] - offs[d*nb]) itself
    std::vector<int64_t> starts((size_t)nparts);
    GSQL_CUDA(ctx, cudaMemcpy2DAsync(starts.data(), 8, offs.p, (size_t)X.nblocks * 8, 8, (size_t)nparts, cudaMemcpyDeviceToHost, ctx->stream));
    GSQL_CUDA(ctx, cudaStreamSynchronize(ctx->stream));
    for (int d = 0; d < nparts; d++) {
        PP.base_row[d] = starts[(size_t)d];
        PP.peer_base[d] = nullptr;  // one address space: the column's address travels in col_off
    }
    for (int c = 0; c < in.n; c++) {
        PP.col_off[c] = (int64_t)(intptr_t)out_data[c];
        PP.null_off[c] = -1;
    }
    {
        KernelScope ks(ctx, "agg_part_scatter");
        switch (in.n) {
        case 1: k_xchg_push_w<true, 1><<<X.nblocks, PW_WARPS * 32, 0, ctx->stream>>>(PP); break;
        case 2: k_xchg_push_w<true, 2><<<X.nblocks, PW_WARPS * 32, 0, ctx->stream>>>(PP); break;
        case 3: k_xchg_push_w<true, 3><<<X.nblocks, PW_WARPS * 32, 0, ctx->stream>>>(PP); break;
        default: k_xchg_push_w<true, 4><<<X.nblocks, PW_WARPS * 32, 0, ctx->stream>>>(PP); break;
        }
    }
    GSQL_CUDA(ctx, cudaGetLastError());
    return GSQL_OK;
}
