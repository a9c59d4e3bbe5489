// NCCL plumbing for captures sharded across the GPUs of one box (SURVEY §8e).
// The exchanges on this path are tiny (chunk statistics, run-carry descriptors, histograms); NVLink bandwidth is
// irrelevant, latency is what counts.  libnccl is dlopen()ed so that
// liburh_b200.so has no link-time dependency on it (single-GPU users never load it) and cannot clash with another
// NCCL copy in the process.
#include "common.cuh"

#include <dlfcn.h>

typedef struct { char internal[128]; } urh_ncclUniqueId;
typedef void* urh_ncclComm_t;
typedef int urh_ncclResult_t;
enum { URH_NCCL_SUM = 0, URH_NCCL_MAX = 2, URH_NCCL_MIN = 3 };
enum { URH_NCCL_UINT8 = 1, URH_NCCL_INT64 = 4, URH_NCCL_FLOAT64 = 8 };

static struct {
    void* handle;
    urh_ncclResult_t (*GetUniqueId)(urh_ncclUniqueId*);
    urh_ncclResult_t (*CommInitRank)(urh_ncclComm_t*, int, urh_ncclUniqueId, int);
    urh_ncclResult_t (*CommDestroy)(urh_ncclComm_t);
    urh_ncclResult_t (*AllReduce)(const void*, void*, size_t, int, int, urh_ncclComm_t, cudaStream_t);
    urh_ncclResult_t (*AllGather)(const void*, void*, size_t, int, urh_ncclComm_t, cudaStream_t);
    urh_ncclResult_t (*Send)(const void*, size_t, int, int, urh_ncclComm_t, cudaStream_t);
    urh_ncclResult_t (*Recv)(void*, size_t, int, int, urh_ncclComm_t, cudaStream_t);
    urh_ncclResult_t (*GroupStart)(void);
    urh_ncclResult_t (*GroupEnd)(void);
    const char* (*GetErrorString)(urh_ncclResult_t);
} g_nccl;

static int nccl_load(char* err, size_t errlen) {
    if (g_nccl.handle) return URH_OK;
    const char* names[] = {getenv("URH_B200_NCCL_LIB"), "libnccl.so.2", "libnccl.so"};
    void* h = nullptr;
    for (const char* n : names) {
        if (!n || !*n) continue;
        h = dlopen(n, RTLD_NOW | RTLD_LOCAL);
        if (h) break;
    }
    if (!h) {
        snprintf(err, errlen, "cannot dlopen libnccl.so.2 (%s)", dlerror());
        return URH_ERR_CUDA;
    }
#define LOADSYM(field, name)                                              \
    *(void**)(&g_nccl.field) = dlsym(h, name);                            \
    if (!g_nccl.field) {                                                  \
        snprintf(err, errlen, "libnccl: missing symbol %s", name);        \
        dlclose(h);                                                       \
        return URH_ERR_CUDA;                                              \
    }
    LOADSYM(GetUniqueId, "ncclGetUniqueId")
    LOADSYM(CommInitRank, "ncclCommInitRank")
    LOADSYM(CommDestroy, "ncclCommDestroy")
    LOADSYM(AllReduce, "ncclAllReduce")
    LOADSYM(AllGather, "ncclAllGather")
    LOADSYM(Send, "ncclSend")
    LOADSYM(Recv, "ncclRecv")
    LOADSYM(GroupStart, "ncclGroupStart")
    LOADSYM(GroupEnd, "ncclGroupEnd")
    LOADSYM(GetErrorString, "ncclGetErrorString")
#undef LOADSYM
    g_nccl.handle = h;
    return URH_OK;
}

#define URH_NCCL(ctx, call)                                                                              \
    do {                                                                                                 \
        urh_ncclResult_t r__ = (call);                                                                   \
        if (r__ != 0) {                                                                                  \
            snprintf((ctx)->err, sizeof((ctx)->err), "%s:%d: %s -> %s", __FILE__, __LINE__, #call,       \
                     g_nccl.GetErrorString ? g_nccl.GetErrorString(r__) : "nccl error");                 \
            return URH_ERR_CUDA;                                                                         \
        }                                                                                                \
    } while (0)

// rank 0 creates the id; the launcher plumbing (torch.distributed / env) broadcasts the 128 bytes
extern "C" int urh_nccl_unique_id(char* out128) {
    char err[256];
    if (nccl_load(err, sizeof(err)) != URH_OK) return URH_ERR_CUDA;
    urh_ncclUniqueId id;
    if (g_nccl.GetUniqueId(&id) != 0) return URH_ERR_CUDA;
    memcpy(out128, id.internal, 128);
    return URH_OK;
}

extern "C" int urh_nccl_init(urh_ctx* ctx, const char* id128, int rank, int world) {
    URH_CHECK(nccl_load(ctx->err, sizeof(ctx->err)));
    URH_CUDA(ctx, cudaSetDevice(ctx->device));
    urh_ncclUniqueId id;
    memcpy(id.internal, id128, 128);
    urh_ncclComm_t comm = nullptr;
    URH_NCCL(ctx, g_nccl.CommInitRank(&comm, world, id, rank));
    ctx->nccl_comm = comm;
    ctx->nccl_rank = rank;
    ctx->nccl_world = world;
    return URH_OK;
}

extern "C" int urh_nccl_destroy(urh_ctx* ctx) {
    if (ctx->nccl_comm && g_nccl.CommDestroy) {
        cudaStreamSynchronize(ctx->stream);
        g_nccl.CommDestroy((urh_ncclComm_t)ctx->nccl_comm);
    }
    ctx->nccl_comm = nullptr;
    ctx->nccl_world = 1;
    ctx->nccl_rank = 0;
    return URH_OK;
}

static int need_comm(urh_ctx* ctx) {
    if (!ctx->nccl_comm) URH_FAIL(ctx, URH_ERR_INVALID, "NCCL communicator not initialised (urh_nccl_init)");
    return URH_OK;
}

// in-place all-reduce on device memory; op: 0 sum, 1 max, 2 min
extern "C" int urh_nccl_allreduce_f64(urh_ctx* ctx, double* d_buf, int64_t count, int op) {
    URH_CHECK(need_comm(ctx));
    const int o = op == 0 ? URH_NCCL_SUM : (op == 1 ? URH_NCCL_MAX : URH_NCCL_MIN);
    URH_NCCL(ctx, g_nccl.AllReduce(d_buf, d_buf, (size_t)count, URH_NCCL_FLOAT64, o, (urh_ncclComm_t)ctx->nccl_comm, ctx->stream));
    return URH_OK;
}
extern "C" int urh_nccl_allreduce_i64(urh_ctx* ctx, int64_t* d_buf, int64_t count, int op) {
    URH_CHECK(need_comm(ctx));
    const int o = op == 0 ? URH_NCCL_SUM : (op == 1 ? URH_NCCL_MAX : URH_NCCL_MIN);
    URH_NCCL(ctx, g_nccl.AllReduce(d_buf, d_buf, (size_t)count, URH_NCCL_INT64, o, (urh_ncclComm_t)ctx->nccl_comm, ctx->stream));
    return URH_OK;
}
// d_recv holds world * bytes_per_rank bytes
extern "C" int urh_nccl_allgather(urh_ctx* ctx, const void* d_send, void* d_recv, size_t bytes_per_rank) {
    URH_CHECK(need_comm(ctx));
    URH_NCCL(ctx, g_nccl.AllGather(d_send, d_recv, bytes_per_rank, URH_NCCL_UINT8, (urh_ncclComm_t)ctx->nccl_comm, ctx->stream));
    return URH_OK;
}

// variable-length gather to `root`: h_bytes[world] are the per-rank byte counts (known to every rank);
// root receives rank r's block at d_recv + sum(h_bytes[0..r))
extern "C" int urh_nccl_gatherv(urh_ctx* ctx, const void* d_send, void* d_recv, const int64_t* h_bytes, int root) {
    URH_CHECK(need_comm(ctx));
    urh_ncclComm_t comm = (urh_ncclComm_t)ctx->nccl_comm;
    URH_NCCL(ctx, g_nccl.GroupStart());
    urh_ncclResult_t bad = 0;
    cudaError_t cbad = cudaSuccess;
    if (ctx->nccl_rank == root) {
        int64_t off = 0;
        for (int r = 0; r < ctx->nccl_world; r++) {
            if (r == root) {
                if (h_bytes[r] > 0) {
                    const cudaError_t e = cudaMemcpyAsync((char*)d_recv + off, d_send, (size_t)h_bytes[r], cudaMemcpyDeviceToDevice, ctx->stream);
                    if (e != cudaSuccess) cbad = e;
                }
            } else if (h_bytes[r] > 0) {
                const urh_ncclResult_t e = g_nccl.Recv((char*)d_recv + off, (size_t)h_bytes[r], URH_NCCL_UINT8, r, comm, ctx->stream);
                if (e != 0) bad = e;
            }
            off += h_bytes[r];
        }
    } else if (h_bytes[ctx->nccl_rank] > 0) {
        bad = g_nccl.Send(d_send, (size_t)h_bytes[ctx->nccl_rank], URH_NCCL_UINT8, root, comm, ctx->stream);
    }
    const urh_ncclResult_t ge = g_nccl.GroupEnd();   // always close the group, then report the first failure
    if (cbad != cudaSuccess) URH_FAIL(ctx, URH_ERR_CUDA, "gatherv: local copy failed: %s", cudaGetErrorString(cbad));
    if (bad != 0) URH_FAIL(ctx, URH_ERR_CUDA, "gatherv: ncclSend/ncclRecv failed: %s", g_nccl.GetErrorString(bad));
    URH_NCCL(ctx, ge);
    return URH_OK;
}

// Grouped point-to-point exchange: send `send_bytes` to `send_peer` and receive `recv_bytes` from `recv_peer` (a peer < 0 or zero
// bytes skips that half).  Used to hand a message that straddles a shard edge to the rank that owns its start.
extern "C" int urh_nccl_sendrecv(urh_ctx* ctx, const void* d_send, size_t send_bytes, int send_peer, void* d_recv, size_t recv_bytes,
                                 int recv_peer) {
    URH_CHECK(need_comm(ctx));
    urh_ncclComm_t comm = (urh_ncclComm_t)ctx->nccl_comm;
    URH_NCCL(ctx, g_nccl.GroupStart());
    urh_ncclResult_t bad = 0;
    if (send_peer >= 0 && send_bytes > 0) {
        const urh_ncclResult_t e = g_nccl.Send(d_send, send_bytes, URH_NCCL_UINT8, send_peer, comm, ctx->stream);
        if (e != 0) bad = e;
    }
    if (recv_peer >= 0 && recv_bytes > 0) {
        const urh_ncclResult_t e = g_nccl.Recv(d_recv, recv_bytes, URH_NCCL_UINT8, recv_peer, comm, ctx->stream);
        if (e != 0) bad = e;
    }
    const urh_ncclResult_t ge = g_nccl.GroupEnd();
    if (bad != 0) URH_FAIL(ctx, URH_ERR_CUDA, "sendrecv: ncclSend/ncclRecv failed: %s", g_nccl.GetErrorString(bad));
    URH_NCCL(ctx, ge);
    return URH_OK;
}

// all-gather of a few host bytes per rank through a device staging buffer (metadata of the sharded digitizer:
// cheaper than a TCP round trip through the launcher's process group)
static int need_stage(urh_ctx* ctx) {
    if (!ctx->nccl_stage) URH_CUDA(ctx, cudaMalloc(&ctx->nccl_stage, 65536));
    if (!ctx->nccl_hstage) URH_CUDA(ctx, cudaHostAlloc(&ctx->nccl_hstage, 65536, cudaHostAllocDefault));
    return URH_OK;
}

extern "C" int urh_nccl_allgather_host(urh_ctx* ctx, const void* h_send, void* h_recv, size_t bytes_per_rank) {
    URH_CHECK(need_comm(ctx));
    URH_CHECK(need_stage(ctx));
    const size_t total = bytes_per_rank * (size_t)ctx->nccl_world;
    const size_t send_pad = (bytes_per_rank + 255) & ~(size_t)255;
    if (send_pad + total > 65536) URH_FAIL(ctx, URH_ERR_INVALID, "allgather_host: payload too large");
    // pinned staging on the host side: the copies are truly asynchronous and the caller's (pageable) buffers are touched
    // by plain memcpy only
    char* d_send = (char*)ctx->nccl_stage;
    char* d_recv = d_send + send_pad;
    char* p_send = (char*)ctx->nccl_hstage;
    char* p_recv = p_send + send_pad;
    memcpy(p_send, h_send, bytes_per_rank);
    URH_CUDA(ctx, cudaMemcpyAsync(d_send, p_send, bytes_per_rank, cudaMemcpyHostToDevice, ctx->stream));
    URH_NCCL(ctx, g_nccl.AllGather(d_send, d_recv, bytes_per_rank, URH_NCCL_UINT8, (urh_ncclComm_t)ctx->nccl_comm, ctx->stream));
    URH_CUDA(ctx, cudaMemcpyAsync(p_recv, d_recv, total, cudaMemcpyDeviceToHost, ctx->stream));
    URH_CUDA(ctx, cudaStreamSynchronize(ctx->stream));
    memcpy(h_recv, p_recv, total);
    return URH_OK;
}

// in-place all-reduce (op: 0 sum, 1 max, 2 min) of a small host int64 array through the same staging buffers
// (the histogram of the capture-wide detect_center: a few thousand bins)
extern "C" int urh_nccl_allreduce_host_i64(urh_ctx* ctx, int64_t* h_buf, int64_t count, int op) {
    URH_CHECK(need_comm(ctx));
    URH_CHECK(need_stage(ctx));
    if (count <= 0) return URH_OK;
    const int o = op == 0 ? URH_NCCL_SUM : (op == 1 ? URH_NCCL_MAX : URH_NCCL_MIN);
    const size_t bytes = (size_t)count * sizeof(int64_t);
    if (bytes <= 65536) {
        memcpy(ctx->nccl_hstage, h_buf, bytes);
        URH_CUDA(ctx, cudaMemcpyAsync(ctx->nccl_stage, ctx->nccl_hstage, bytes, cudaMemcpyHostToDevice, ctx->stream));
        URH_NCCL(ctx, g_nccl.AllReduce(ctx->nccl_stage, ctx->nccl_stage, (size_t)count, URH_NCCL_INT64, o, (urh_ncclComm_t)ctx->nccl_comm, ctx->stream));
        URH_CUDA(ctx, cudaMemcpyAsync(ctx->nccl_hstage, ctx->nccl_stage, bytes, cudaMemcpyDeviceToHost, ctx->stream));
        URH_CUDA(ctx, cudaStreamSynchronize(ctx->stream));
        memcpy(h_buf, ctx->nccl_hstage, bytes);
        return URH_OK;
    }
    int64_t* d = nullptr;
    URH_CUDA(ctx, cudaMallocAsync((void**)&d, bytes, ctx->stream));
    URH_CUDA(ctx, cudaMemcpyAsync(d, h_buf, bytes, cudaMemcpyHostToDevice, ctx->stream));
    URH_NCCL(ctx, g_nccl.AllReduce(d, d, (size_t)count, URH_NCCL_INT64, o, (urh_ncclComm_t)ctx->nccl_comm, ctx->stream));
    URH_CUDA(ctx, cudaMemcpyAsync(h_buf, d, bytes, cudaMemcpyDeviceToHost, ctx->stream));
    URH_CUDA(ctx, cudaFreeAsync(d, ctx->stream));
    URH_CUDA(ctx, cudaStreamSynchronize(ctx->stream));
    return URH_OK;
}
