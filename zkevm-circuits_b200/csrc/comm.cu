// comm.cu -- communicator of a context for the multi-GPU create_proof and the sharded NTT / MSM.
//
// The proving session stays replicated (every rank runs the same host code on the same inputs and therefore produces
// the same transcript and the same proof bytes); independent units -- columns, lookup arguments, permutation sets, the
// quotient's coset parts, the evaluations of one rotation -- are cut into P contiguous blocks (rank r computes block r, see
// prover.cu's Deal) and each result is completed by ONE in-place all-gather: every rank contributes its own block of a slab.
// A single commitment is sharded by point range instead, its 64-byte partial sums all-gathered and added on the host.
//
// Two backends implement the same five primitives (comm_allgather, comm_alltoall, comm_allreduce_u64, comm_barrier, comm_window):
//   NCCL (zkb_comm_init): one process per GPU; NCCL is resolved at run time (dlopen of libnccl.so.2: inside a torch process that
//        is torch's bundled copy); the exchange window is a cudaIpc-mapped block per rank.
//   in-process (zkb_comm_init_local): P contexts of ONE process on one device, each driven from its own host thread, so that the
//        whole multi-rank path runs on a single GPU.  Stream-ordered like NCCL: a rank records an event on its stream and meets
//        the others on the host, then makes its stream wait on every peer's event and copies the peer blocks device-to-device;
//        a second meeting (again with events) keeps a rank from overwriting its send block before every peer has copied it.
//        Every collective carries its kind and byte count, checked at the first meeting; a disagreement or a meeting that
//        waits longer than the group's timeout poisons the group, and every later collective fails at once.
#include "common.cuh"
#include <dlfcn.h>
#include <nccl.h>
#include <string.h>
#include <chrono>
#include <condition_variable>
#include <mutex>

namespace zkb {

struct NcclApi {
    void *handle = nullptr;
    ncclResult_t (*GetUniqueId)(ncclUniqueId *) = nullptr;
    ncclResult_t (*CommInitRank)(ncclComm_t *, int, ncclUniqueId, int) = nullptr;
    ncclResult_t (*CommDestroy)(ncclComm_t) = nullptr;
    ncclResult_t (*AllReduce)(const void *, void *, size_t, ncclDataType_t, ncclRedOp_t, ncclComm_t, cudaStream_t) = nullptr;
    ncclResult_t (*AllGather)(const void *, void *, size_t, ncclDataType_t, ncclComm_t, cudaStream_t) = nullptr;
    ncclResult_t (*Send)(const void *, size_t, ncclDataType_t, int, ncclComm_t, cudaStream_t) = nullptr;
    ncclResult_t (*Recv)(void *, size_t, ncclDataType_t, int, ncclComm_t, cudaStream_t) = nullptr;
    ncclResult_t (*GroupStart)() = nullptr;
    ncclResult_t (*GroupEnd)() = nullptr;
    const char *(*GetErrorString)(ncclResult_t) = nullptr;
};

struct NcclLoad {
    NcclApi api;
    bool ok = false;
    char err[256] = "";
};

// resolved once: a function-local static is initialised exactly once even when several threads ask for it together
static NcclApi *nccl_api() {
    static NcclLoad *const L = []() {
        NcclLoad *l = new NcclLoad();
        NcclApi &api = l->api;
        void *h = dlopen("libnccl.so.2", RTLD_NOW | RTLD_GLOBAL);
        if (!h) h = dlopen("libnccl.so", RTLD_NOW | RTLD_GLOBAL);
        if (!h) { snprintf(l->err, sizeof(l->err), "cannot load libnccl.so.2: %s", dlerror()); return l; }
        api.GetUniqueId = (decltype(api.GetUniqueId))dlsym(h, "ncclGetUniqueId");
        api.CommInitRank = (decltype(api.CommInitRank))dlsym(h, "ncclCommInitRank");
        api.CommDestroy = (decltype(api.CommDestroy))dlsym(h, "ncclCommDestroy");
        api.AllReduce = (decltype(api.AllReduce))dlsym(h, "ncclAllReduce");
        api.GetErrorString = (decltype(api.GetErrorString))dlsym(h, "ncclGetErrorString");
        api.AllGather = (decltype(api.AllGather))dlsym(h, "ncclAllGather");
        api.Send = (decltype(api.Send))dlsym(h, "ncclSend");
        api.Recv = (decltype(api.Recv))dlsym(h, "ncclRecv");
        api.GroupStart = (decltype(api.GroupStart))dlsym(h, "ncclGroupStart");
        api.GroupEnd = (decltype(api.GroupEnd))dlsym(h, "ncclGroupEnd");
        if (!api.GetUniqueId || !api.CommInitRank || !api.CommDestroy || !api.AllReduce || !api.AllGather || !api.Send || !api.Recv || !api.GroupStart || !api.GroupEnd) {
            snprintf(l->err, sizeof(l->err), "libnccl.so.2 lacks required symbols");
            return l;
        }
        api.handle = h;
        l->ok = true;
        return l;
    }();
    if (!L->ok) { set_error("%s", L->err); return nullptr; }
    return &L->api;
}

#define ZKB_NCCL(api, expr)                                                                                           \
    do {                                                                                                              \
        ncclResult_t _r = (expr);                                                                                     \
        if (_r != ncclSuccess) {                                                                                      \
            zkb::set_error("%s:%d NCCL: %s", __FILE__, __LINE__, (api)->GetErrorString ? (api)->GetErrorString(_r) : "error"); \
            return ZKB_ERR_CUDA;                                                                                      \
        }                                                                                                             \
    } while (0)

// ---- in-process backend ------------------------------------------------------------------------------------------------------
enum LocalKind { LK_ALLGATHER = 1, LK_ALLTOALL = 2, LK_ALLREDUCE_U64 = 3 };
static const char *local_kind_name(int k) {
    return k == LK_ALLGATHER ? "all-gather" : k == LK_ALLTOALL ? "all-to-all" : k == LK_ALLREDUCE_U64 ? "u64 all-reduce" : "?";
}

struct LocalGroup {
    int P = 0;
    uint32_t timeout_ms = 0;
    std::mutex mu;
    std::condition_variable cv;
    uint64_t meetings = 0;   // completed meetings
    int arrived = 0;         // ranks waiting in the current meeting
    int members = 0;         // contexts still joined
    bool poisoned = false;
    char why[320] = "";
    struct Post {            // what rank r brought to the current collective (written before its first meeting)
        int kind = 0;
        size_t bytes = 0;
        uint64_t seq = 0;
        const void *send = nullptr;
    } post[16];
    cudaEvent_t ready[16] = {}, done[16] = {};   // rank r's send block is written / rank r has copied every peer block
};

struct LocalRank {
    LocalGroup *g = nullptr;
    uint64_t seq = 0;              // collectives this rank has entered
    uint64_t *staging = nullptr;   // the all-reduce's P blocks
    size_t staging_bytes = 0;
};

// all ranks meet on the host.  Called with the group's lock held; fails (the group poisoned) when the meeting outlasts the timeout
static int32_t local_meet(LocalGroup *g, std::unique_lock<std::mutex> &lk, int rank, uint64_t seq) {
    const uint64_t mine = g->meetings;
    if (++g->arrived == g->P) {
        g->arrived = 0;
        g->meetings++;
        g->cv.notify_all();
        return ZKB_OK;
    }
    g->cv.wait_for(lk, std::chrono::milliseconds(g->timeout_ms), [&] { return g->meetings != mine || g->poisoned; });
    if (g->meetings != mine) return ZKB_OK;
    if (!g->poisoned) {
        g->poisoned = true;
        snprintf(g->why, sizeof(g->why), "rank %d waited more than %u ms for the other ranks at collective #%llu", rank, g->timeout_ms,
                 (unsigned long long)seq);
        g->cv.notify_all();
    }
    set_error("in-process communicator: %s", g->why);
    return ZKB_ERR_STATE;
}

__global__ void sum_u64_kernel(const uint64_t *__restrict__ blocks, int P, size_t count, uint64_t *__restrict__ out) {
    const size_t i = blockIdx.x * (size_t)blockDim.x + threadIdx.x;
    if (i >= count) return;
    uint64_t s = 0;
    for (int j = 0; j < P; ++j) s += blocks[(size_t)j * count + i];
    out[i] = s;
}

// one collective of the in-process group.  all-gather: rank j's `bytes` at send -> recv block j.  all-to-all: block r of rank j's
// send -> recv block j.  all-reduce: every rank's `bytes` at send (= recv) -> staging block j, then the sum into recv.
static int32_t local_collective(zkb_ctx *ctx, int kind, const void *send, void *recv, size_t bytes, cudaStream_t st) {
    LocalRank *me = (LocalRank *)ctx->local_comm;
    LocalGroup *g = me->g;
    const int P = g->P, r = ctx->rank;
    const uint64_t seq = me->seq++;
    uint8_t *dst = (uint8_t *)recv;
    if (kind == LK_ALLREDUCE_U64) {
        if (me->staging_bytes < bytes * P) {
            if (me->staging) { ZKB_CUDA(cudaStreamSynchronize(st)); ZKB_CUDA(cudaFree(me->staging)); me->staging = nullptr; me->staging_bytes = 0; }
            ZKB_CUDA(cudaMalloc((void **)&me->staging, bytes * P));
            me->staging_bytes = bytes * P;
        }
        dst = (uint8_t *)me->staging;
    }
    const void *peer_send[16];
    {
        std::unique_lock<std::mutex> lk(g->mu);
        if (g->poisoned) { set_error("in-process communicator: %s", g->why); return ZKB_ERR_STATE; }
        // every peer queued its wait on this event in the previous collective before the second meeting, which this rank has passed
        ZKB_CUDA(cudaEventRecord(g->ready[r], st));
        g->post[r].kind = kind;
        g->post[r].bytes = bytes;
        g->post[r].seq = seq;
        g->post[r].send = send;
        ZKB_TRY(local_meet(g, lk, r, seq));
        // the same collective everywhere, or nothing is queued: every rank sees the same posts and fails the same way
        for (int j = 0; j < P; ++j) {
            const LocalGroup::Post &a = g->post[0], &b = g->post[j];
            if (a.kind != b.kind || a.bytes != b.bytes || a.seq != b.seq) {
                char msg[320];
                snprintf(msg, sizeof(msg), "ranks disagree at collective #%llu: rank 0 called %s of %zu bytes (its collective #%llu), rank %d called %s of "
                         "%zu bytes (its collective #%llu)", (unsigned long long)seq, local_kind_name(a.kind), a.bytes, (unsigned long long)a.seq, j,
                         local_kind_name(b.kind), b.bytes, (unsigned long long)b.seq);
                if (!g->poisoned) { g->poisoned = true; snprintf(g->why, sizeof(g->why), "%s", msg); g->cv.notify_all(); }
                set_error("in-process communicator: %s", msg);
                return ZKB_ERR_STATE;
            }
            peer_send[j] = b.send;
        }
    }
    for (int j = 0; j < P; ++j) {
        const uint8_t *src = (const uint8_t *)peer_send[j] + (kind == LK_ALLTOALL ? (size_t)r * bytes : 0);
        if (j != r) ZKB_CUDA(cudaStreamWaitEvent(st, g->ready[j], 0));
        if (src != dst + (size_t)j * bytes) ZKB_CUDA(cudaMemcpyAsync(dst + (size_t)j * bytes, src, bytes, cudaMemcpyDeviceToDevice, st));
    }
    {
        std::unique_lock<std::mutex> lk(g->mu);
        ZKB_CUDA(cudaEventRecord(g->done[r], st));
        ZKB_TRY(local_meet(g, lk, r, seq));
    }
    // later work on this stream may overwrite the send block: after every peer's copies out of it
    for (int j = 0; j < P; ++j)
        if (j != r) ZKB_CUDA(cudaStreamWaitEvent(st, g->done[j], 0));
    if (kind == LK_ALLREDUCE_U64) {
        const size_t count = bytes / 8;
        sum_u64_kernel<<<(unsigned)((count + 127) / 128), 128, 0, st>>>(me->staging, P, count, (uint64_t *)recv);
        ctx->launches++;
        ZKB_CUDA(cudaGetLastError());
    }
    return ZKB_OK;
}

// in-place sum of `count` u64 words on the device (disjoint supports -> exact gather)
int32_t comm_allreduce_u64(zkb_ctx *ctx, void *dev_buf, size_t count, cudaStream_t st) {
    if (ctx->nranks <= 1) return ZKB_OK;
    if (ctx->local_comm) return local_collective(ctx, LK_ALLREDUCE_U64, dev_buf, dev_buf, count * 8, st);
    NcclApi *api = nccl_api();
    if (!api || !ctx->nccl_comm) { set_error("communicator not initialised"); return ZKB_ERR_STATE; }
    ZKB_NCCL(api, api->AllReduce(dev_buf, dev_buf, count, ncclUint64, ncclSum, (ncclComm_t)ctx->nccl_comm, st));
    return ZKB_OK;
}

int32_t comm_allgather(zkb_ctx *ctx, const void *send, void *recv, size_t bytes_per_rank, cudaStream_t st) {
    if (ctx->nranks <= 1) {
        if (send != recv) ZKB_CUDA(cudaMemcpyAsync(recv, send, bytes_per_rank, cudaMemcpyDeviceToDevice, st));
        return ZKB_OK;
    }
    if (ctx->local_comm) return local_collective(ctx, LK_ALLGATHER, send, recv, bytes_per_rank, st);
    NcclApi *api = nccl_api();
    if (!api || !ctx->nccl_comm) { set_error("communicator not initialised"); return ZKB_ERR_STATE; }
    ZKB_NCCL(api, api->AllGather(send, recv, bytes_per_rank, ncclUint8, (ncclComm_t)ctx->nccl_comm, st));
    return ZKB_OK;
}

int32_t comm_alltoall(zkb_ctx *ctx, const void *send, void *recv, size_t bytes_per_block, cudaStream_t st) {
    if (ctx->nranks <= 1) {
        if (send != recv) ZKB_CUDA(cudaMemcpyAsync(recv, send, bytes_per_block, cudaMemcpyDeviceToDevice, st));
        return ZKB_OK;
    }
    if (ctx->local_comm) return local_collective(ctx, LK_ALLTOALL, send, recv, bytes_per_block, st);
    NcclApi *api = nccl_api();
    if (!api || !ctx->nccl_comm) { set_error("communicator not initialised"); return ZKB_ERR_STATE; }
    ncclComm_t comm = (ncclComm_t)ctx->nccl_comm;
    ZKB_NCCL(api, api->GroupStart());
    for (int j = 0; j < ctx->nranks; ++j) {
        ZKB_NCCL(api, api->Send((const uint8_t *)send + (size_t)j * bytes_per_block, bytes_per_block, ncclUint8, j, comm, st));
        ZKB_NCCL(api, api->Recv((uint8_t *)recv + (size_t)j * bytes_per_block, bytes_per_block, ncclUint8, j, comm, st));
    }
    ZKB_NCCL(api, api->GroupEnd());
    return ZKB_OK;
}

int32_t comm_barrier(zkb_ctx *ctx, cudaStream_t st) {
    if (ctx->nranks <= 1) return ZKB_OK;
    void *w = nullptr;
    ZKB_TRY(scratch_get(ctx, SCR_COMM_FLAG, 64, &w));
    return comm_allreduce_u64(ctx, w, 1, st);
}

// Exchange window: one cudaMalloc block per rank, mapped by every other rank; afterwards ctx->win_peers[j] is a pointer that
// kernels on THIS device can load from / store to.  NCCL backend: the block is exported with cudaIpcGetMemHandle, the 64-byte
// handles are all-gathered and opened by every other rank (cudaIpcMemLazyEnablePeerAccess), so the traffic goes over NVLink /
// NVSwitch as plain peer accesses.  In-process backend: the ranks share one device and one address space, so the all-gathered
// 64-byte record carries the block's pointer itself and nothing is opened or closed.
int32_t comm_window(zkb_ctx *ctx, size_t bytes, cudaStream_t st) {
    if (ctx->win_bytes >= bytes && ctx->win_local) return ZKB_OK;
    const bool ipc = ctx->local_comm == nullptr;
    // every rank must be past its last use of the old windows before anyone unmaps them
    ZKB_TRY(comm_barrier(ctx, st));
    ZKB_CUDA(cudaStreamSynchronize(st));
    for (int j = 0; j < ctx->nranks; ++j)
        if (j != ctx->rank && ctx->win_peers[j]) { if (ipc) cudaIpcCloseMemHandle(ctx->win_peers[j]); ctx->win_peers[j] = nullptr; }
    if (ctx->nranks > 1) { ZKB_TRY(comm_barrier(ctx, st)); ZKB_CUDA(cudaStreamSynchronize(st)); }   // all peers unmapped before the owner frees
    if (ctx->win_local) { ZKB_CUDA(cudaFree(ctx->win_local)); ctx->win_local = nullptr; ctx->win_bytes = 0; }
    const size_t want = (bytes + (2u << 20) - 1) & ~(size_t)((2u << 20) - 1);
    ZKB_CUDA(cudaMalloc(&ctx->win_local, want));
    ctx->win_bytes = want;
    ctx->win_peers[ctx->rank] = ctx->win_local;
    if (ctx->nranks <= 1) return ZKB_OK;
    static_assert(sizeof(cudaIpcMemHandle_t) == 64, "cudaIpcMemHandle_t is 64 bytes");
    cudaIpcMemHandle_t mine;
    memset(&mine, 0, sizeof(mine));
    if (ipc) ZKB_CUDA(cudaIpcGetMemHandle(&mine, ctx->win_local));
    else memcpy(&mine, &ctx->win_local, sizeof(void *));
    uint8_t *d_h = nullptr;
    ZKB_TRY(scratch_get(ctx, SCR_COMM, 64 * 16, (void **)&d_h));
    ZKB_CUDA(cudaMemcpyAsync(d_h + 64 * ctx->rank, &mine, 64, cudaMemcpyHostToDevice, st));
    ZKB_TRY(comm_allgather(ctx, d_h + 64 * ctx->rank, d_h, 64, st));
    cudaIpcMemHandle_t all[16];
    ZKB_CUDA(cudaMemcpyAsync(all, d_h, 64 * (size_t)ctx->nranks, cudaMemcpyDeviceToHost, st));
    ZKB_CUDA(cudaStreamSynchronize(st));
    for (int j = 0; j < ctx->nranks; ++j) {
        if (j == ctx->rank) continue;
        if (ipc) ZKB_CUDA(cudaIpcOpenMemHandle(&ctx->win_peers[j], all[j], cudaIpcMemLazyEnablePeerAccess));
        else memcpy(&ctx->win_peers[j], &all[j], sizeof(void *));
    }
    return ZKB_OK;
}

}  // namespace zkb
using namespace zkb;

extern "C" int32_t zkb_comm_unique_id(uint8_t out[128]) {
    ZKB_ARG(out != nullptr);
    NcclApi *api = nccl_api();
    if (!api) return ZKB_ERR_CUDA;
    ncclUniqueId id;
    static_assert(sizeof(ncclUniqueId) == 128, "ncclUniqueId is 128 bytes");
    ZKB_NCCL(api, api->GetUniqueId(&id));
    memcpy(out, &id, 128);
    return ZKB_OK;
}

extern "C" int32_t zkb_comm_init(zkb_ctx *ctx, const uint8_t unique_id[128], int32_t rank, int32_t nranks) {
    // at most 16 ranks: win_peers, the exchange routes and the SCR_COMM records hold 16 entries
    ZKB_ARG(ctx && unique_id && nranks >= 1 && nranks <= 16 && rank >= 0 && rank < nranks);
    if (ctx->nccl_comm || ctx->local_comm) { set_error("communicator already initialised"); return ZKB_ERR_STATE; }
    ZKB_CUDA(cudaSetDevice(ctx->device));
    NcclApi *api = nccl_api();
    if (!api) return ZKB_ERR_CUDA;
    ncclUniqueId id;
    memcpy(&id, unique_id, 128);
    ncclComm_t comm = nullptr;
    ZKB_NCCL(api, api->CommInitRank(&comm, nranks, id, rank));
    ctx->nccl_comm = comm;
    ctx->rank = rank;
    ctx->nranks = nranks;
    return ZKB_OK;
}

extern "C" int32_t zkb_comm_init_local(zkb_ctx *const *ctxs, int32_t nranks, uint32_t timeout_ms) {
    ZKB_ARG(ctxs && nranks >= 1 && nranks <= 16 && timeout_ms > 0);
    for (int i = 0; i < nranks; ++i) {
        ZKB_ARG(ctxs[i]);
        if (ctxs[i]->device != ctxs[0]->device) { set_error("context %d is on device %d, context 0 on device %d: one device per group", i, ctxs[i]->device, ctxs[0]->device); return ZKB_ERR_ARG; }
        if (ctxs[i]->nccl_comm || ctxs[i]->local_comm) { set_error("context %d already has a communicator", i); return ZKB_ERR_ARG; }
        for (int j = 0; j < i; ++j)
            if (ctxs[j] == ctxs[i]) { set_error("contexts %d and %d are the same context", j, i); return ZKB_ERR_ARG; }
    }
    ZKB_CUDA(cudaSetDevice(ctxs[0]->device));
    LocalGroup *g = new LocalGroup();
    g->P = nranks;
    g->timeout_ms = timeout_ms;
    for (int i = 0; i < nranks; ++i) {
        cudaError_t e = cudaEventCreateWithFlags(&g->ready[i], cudaEventDisableTiming);
        if (e == cudaSuccess) e = cudaEventCreateWithFlags(&g->done[i], cudaEventDisableTiming);
        if (e != cudaSuccess) {
            for (int j = 0; j <= i; ++j) { if (g->ready[j]) cudaEventDestroy(g->ready[j]); if (g->done[j]) cudaEventDestroy(g->done[j]); }
            delete g;
            set_error("cudaEventCreate: %s", cudaGetErrorString(e));
            return ZKB_ERR_CUDA;
        }
    }
    g->members = nranks;
    for (int i = 0; i < nranks; ++i) {
        LocalRank *me = new LocalRank();
        me->g = g;
        ctxs[i]->local_comm = me;
        ctxs[i]->rank = i;
        ctxs[i]->nranks = nranks;
    }
    return ZKB_OK;
}

extern "C" int32_t zkb_comm_destroy(zkb_ctx *ctx) {
    ZKB_ARG(ctx);
    // exchange window: unmap the peers' blocks, free the own one (the peers close their mappings in their own destroy)
    for (int j = 0; j < 16; ++j)
        if (j != ctx->rank && ctx->win_peers[j]) { if (!ctx->local_comm) cudaIpcCloseMemHandle(ctx->win_peers[j]); ctx->win_peers[j] = nullptr; }
    if (ctx->nccl_comm) {
        NcclApi *api = nccl_api();
        cudaStreamSynchronize(ctx->stream);
        if (api) api->CommDestroy((ncclComm_t)ctx->nccl_comm);
        ctx->nccl_comm = nullptr;
    }
    if (ctx->local_comm) {
        LocalRank *me = (LocalRank *)ctx->local_comm;
        LocalGroup *g = me->g;
        cudaStreamSynchronize(ctx->stream);
        bool last;
        {
            // a rank that leaves ends the group: the others' next collective fails at once instead of waiting for it
            std::lock_guard<std::mutex> lk(g->mu);
            if (!g->poisoned) { g->poisoned = true; snprintf(g->why, sizeof(g->why), "rank %d has left the group", ctx->rank); }
            g->cv.notify_all();
            last = --g->members == 0;
        }
        if (me->staging) cudaFree(me->staging);
        delete me;
        if (last) {
            for (int j = 0; j < g->P; ++j) { cudaEventDestroy(g->ready[j]); cudaEventDestroy(g->done[j]); }
            delete g;
        }
        ctx->local_comm = nullptr;
    }
    if (ctx->win_local) { cudaFree(ctx->win_local); ctx->win_local = nullptr; ctx->win_bytes = 0; }
    ctx->win_peers[ctx->rank] = nullptr;
    for (auto &kv : ctx->shard_tw) cudaFree(kv.second);
    ctx->shard_tw.clear();
    ctx->rank = 0;
    ctx->nranks = 1;
    return ZKB_OK;
}
