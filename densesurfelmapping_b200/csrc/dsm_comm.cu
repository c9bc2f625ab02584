// Multi-GPU side of the C ABI (include/dsm.h "multi-GPU"): one context per GPU (one process or thread each), frames of a
// batch sharded across the contexts, and ONE gather of the per-GPU surfel deltas onto a root rank at the end of a batch
// (SURVEY.md section 8e; BASELINE configs[3]).  The reference has no counterpart: fuse_initialize_map is single-process
// (fusion_functions.cpp:30-83); what travels is what SurfelMap::fuse_map consumes after the call (surfel_map.cpp:1077-1109):
// the new surfels and the updated local surfels of every frame.
//
// Wire format of one rank's payload (little endian; tests/ and densesurfelmapping_b200/gather.py restate it):
//   int32  magic 'DSMD', n_frames, n_new_total, n_pool_total
//   int32  n_new[n_frames]
//   int32  pool_ofs[n_frames + 1]
//   pad to a multiple of 16 bytes
//   dsm_surfel_t new[n_new_total]     valid new surfels only, frame by frame, seed-index order (fusion_functions.cpp:320-359)
//   dsm_surfel_t pool[n_pool_total]   the frames' updated local surfels, batch order
// Two transports, same wire format:
//  * ranks on one node (the normal case: NVLink / NVSwitch peers) -- ONE-SIDED WRITES OVER PEER MEMORY.  The root's
//    receive buffer (one capacity-sized slot per rank) and a small control block are shared with the other processes by
//    CUDA IPC once (handles exchanged with ncclAllGather at the first gather); from then on a gather is a pack kernel on
//    every rank that writes its header, its valid new surfels and its pool straight into its slot in the ROOT's memory
//    (coalesced peer stores), followed by a release-store of the gather's sequence number.  Nothing waits on the host:
//    the counts stay on the device, exactly the valid bytes cross NVLink, no NCCL kernel runs per step.  Flow control is
//    a credit the root publishes when it enters the gather (a sender's pack waits for it on the device); completion is
//    observed by the root's HOST in dsm_gather_wait (it polls the control block through a stream of its own), so no kernel
//    of the root ever spins on its peers.
//  * otherwise (no peer mapping, or DSM_GATHER_NCCL=1) -- NCCL: counts to the host, ncclAllGather of the byte counts,
//    one grouped ncclSend / ncclRecv.
// Only valid records travel (the padded [n_frames][S] new-surfel buffer never does).  Counts must be known on the host
// to size the messages, so the call waits for the batch's kernels once (new-surfel counts to pinned memory), then
// packs on a side stream (the next batch's kernels may start as soon as the pack has read the buffers), exchanges the
// byte counts with one ncclAllGather and moves the payloads with one grouped ncclSend / ncclRecv.
//
// NCCL is loaded at run time (dlopen "libnccl.so.2": inside a PyTorch process that is the NCCL torch already loaded,
// in a plain C++ process the system one), so the library has no link-time dependency on it.
#include "dsm_ctx.hpp"
#include <cstring>
#include <new>
#include <dlfcn.h>
#include <unistd.h>
#include <vector>
#include <nccl.h>

struct DsmNccl
{
    void *lib = nullptr;
    decltype(&ncclGetUniqueId) GetUniqueId = nullptr;
    decltype(&ncclCommInitRank) CommInitRank = nullptr;
    decltype(&ncclCommDestroy) CommDestroy = nullptr;
    decltype(&ncclAllGather) AllGather = nullptr;
    decltype(&ncclSend) Send = nullptr;
    decltype(&ncclRecv) Recv = nullptr;
    decltype(&ncclGroupStart) GroupStart = nullptr;
    decltype(&ncclGroupEnd) GroupEnd = nullptr;
    decltype(&ncclGetErrorString) GetErrorString = nullptr;
};

static DsmNccl *nccl_api()
{
    static DsmNccl api;
    static bool tried = false;
    if (tried) return api.lib ? &api : nullptr;
    tried = true;
    void *h = dlopen("libnccl.so.2", RTLD_NOW | RTLD_LOCAL);
    if (!h) h = dlopen("libnccl.so", RTLD_NOW | RTLD_LOCAL);
    if (!h) return nullptr;
#define SYM(field, name)                                        \
    api.field = (decltype(api.field))dlsym(h, name);            \
    if (!api.field) return nullptr;
    SYM(GetUniqueId, "ncclGetUniqueId")
    SYM(CommInitRank, "ncclCommInitRank")
    SYM(CommDestroy, "ncclCommDestroy")
    SYM(AllGather, "ncclAllGather")
    SYM(Send, "ncclSend")
    SYM(Recv, "ncclRecv")
    SYM(GroupStart, "ncclGroupStart")
    SYM(GroupEnd, "ncclGroupEnd")
    SYM(GetErrorString, "ncclGetErrorString")
#undef SYM
    api.lib = h;
    return &api;
}

struct DsmComm
{
    CudaOwner own; // the buffers, streams and events below, except recv
    ncclComm_t comm = nullptr;
    int rank = 0, nranks = 1;
    cudaStream_t stream = nullptr;       // pack + collectives
    cudaEvent_t ev_kernels = nullptr;    // the batch's kernels have finished (counts readable)
    cudaEvent_t ev_packed = nullptr;     // the pack has read newsurf / pool: the next batch may overwrite them
    unsigned char *pack = nullptr;       // device: this rank's payload
    size_t pack_cap = 0;
    DevPtr<unsigned char> recv;          // device, root only: all payloads back to back (grown on demand)
    size_t recv_cap = 0;
    int64_t *d_bytes = nullptr;          // device [nranks]
    int64_t *h_bytes = nullptr;          // pinned [nranks]
    int32_t *h_cnt = nullptr;            // pinned [max_batch]: new-surfel counts of the batch (NCCL transport)
    std::vector<size_t> ofs;             // root: byte offset of every rank's payload in recv (nranks + 1)
    int last_root = -1;
    // ---- peer-memory transport
    bool force_nccl = false;             // DSM_GATHER_NCCL=1
    int peer_root = -1;                  // root the mapping below was made for (-1: none yet)
    bool peer_ok = false;                // every rank mapped the root's buffers
    size_t slot_bytes = 0;               // capacity of one rank's slot (payload_cap rounded up to 256)
    unsigned char *slots = nullptr;      // local allocation: nranks slots (used when this rank is the root)
    struct DsmPeerCtrl *ctrl = nullptr;  // local allocation: control block (used when this rank is the root)
    unsigned char *r_slots = nullptr;    // the ROOT's slots as seen from this rank (== slots on the root)
    struct DsmPeerCtrl *r_ctrl = nullptr;
    std::unique_ptr<void, Release<void *, cudaIpcCloseMemHandle>> ipc_slots, ipc_ctrl; // other ranks: what r_slots / r_ctrl map
    unsigned long long seq = 0;          // gathers done on this mapping
    unsigned char *d_handles = nullptr;  // device staging for the handle exchange [nranks][128]
    bool last_peer = false;              // the last gather used the peer transport
    cudaStream_t poll = nullptr;         // root: reads the control block while the side stream is busy
    unsigned long long *h_arrived = nullptr; // pinned [DSM_MAX_RANKS]
    unsigned long long done_seq = 0;     // root: every payload of gathers <= done_seq has been seen complete
};

#define DSM_MAX_RANKS 64
struct DsmPeerCtrl
{
    unsigned long long arrived[DSM_MAX_RANKS]; // sequence number of the last gather whose payload of rank r is complete
    long long bytes[DSM_MAX_RANKS];            // its size
    unsigned long long credit;                 // sequence number of the gather the root is ready to receive
};

#define NK(call)                                                                                                  \
    do                                                                                                            \
    {                                                                                                             \
        ncclResult_t _r = (call);                                                                                 \
        if (_r != ncclSuccess)                                                                                    \
        {                                                                                                         \
            snprintf(ctx->err, sizeof(ctx->err), "%s:%d %s -> %s", __FILE__, __LINE__, #call, api->GetErrorString(_r)); \
            return DSM_E_NCCL;                                                                                    \
        }                                                                                                         \
    } while (0)

static size_t header_bytes(int n_frames) { return ((size_t)(4 + n_frames + n_frames + 1) * 4 + 15) / 16 * 16; }
static size_t payload_cap(const dsm_ctx *ctx)
{
    return header_bytes(ctx->p.max_batch) + ((size_t)ctx->p.max_batch * ctx->d.S + (size_t)(ctx->p.max_local_surfels > 0 ? ctx->p.max_local_surfels : 1)) * sizeof(dsm_surfel_t);
}

// ---- peer-memory transport: device side ----
__device__ __forceinline__ unsigned long long ld_acquire_sys(const unsigned long long *p)
{
    unsigned long long v;
    asm volatile("ld.acquire.sys.global.u64 %0, [%1];" : "=l"(v) : "l"(p) : "memory");
    return v;
}
__device__ __forceinline__ void st_release_sys(unsigned long long *p, unsigned long long v)
{
    asm volatile("st.release.sys.global.u64 [%0], %1;" ::"l"(p), "l"(v) : "memory");
}
// bounded device-side wait (about 20 s): a peer that never arrives traps instead of hanging the GPU
#define DSM_SPIN_LIMIT (1u << 26)

__global__ void k_peer_credit(DsmPeerCtrl *ctrl, unsigned long long seq) { st_release_sys(&ctrl->credit, seq); }

__global__ void k_peer_wait_credit(const DsmPeerCtrl *ctrl, unsigned long long seq)
{
    unsigned spin = 0;
    while (ld_acquire_sys(&ctrl->credit) < seq)
    {
        __nanosleep(256);
        if (++spin > DSM_SPIN_LIMIT) __trap();
    }
}

// One rank's payload, the only writer of the wire format: straight into its slot in the root's memory (peer transport) or
// into the local send buffer (NCCL).  blockIdx.y < nb -> the valid new surfels of frame blockIdx.y, blockIdx.y == nb ->
// the pool and (block 0) the header.  4-byte words, coalesced.
__global__ void __launch_bounds__(256) k_peer_pack(const dsm_surfel_t *newsurf, const int32_t *nnew, const dsm_surfel_t *pool,
                                                   const int32_t *poolofs, int S, int nb, unsigned char *slot, unsigned hb)
{
    const int f = blockIdx.y;
    int before = 0, total = 0;
    for (int i = 0; i < nb; i++)
    { // nb <= max_batch: a few dozen adds
        const int c = nnew[i];
        if (i < f) before += c;
        total += c;
    }
    const int stride = gridDim.x * blockDim.x, t0 = blockIdx.x * blockDim.x + threadIdx.x;
    uint32_t *body = reinterpret_cast<uint32_t *>(slot + hb);
    if (f < nb)
    {
        const int n = nnew[f];
        const uint32_t *src = reinterpret_cast<const uint32_t *>(newsurf + (size_t)f * S);
        uint32_t *dst = body + (size_t)before * 11;
        for (int w = t0; w < n * 11; w += stride) dst[w] = src[w];
        return;
    }
    const int n_pool = poolofs[nb];
    const uint32_t *src = reinterpret_cast<const uint32_t *>(pool);
    uint32_t *dst = body + (size_t)total * 11;
    for (size_t w = t0; w < (size_t)n_pool * 11; w += stride) dst[w] = src[w];
    if (blockIdx.x == 0)
    {
        int32_t *h = reinterpret_cast<int32_t *>(slot);
        const int hw = (int)(hb / 4);
        for (int i = threadIdx.x; i < hw; i += blockDim.x)
        {
            int32_t v = 0;
            if (i == 0) v = 0x444d5344; // 'DSMD'
            else if (i == 1) v = nb;
            else if (i == 2) v = total;
            else if (i == 3) v = n_pool;
            else if (i < 4 + nb) v = nnew[i - 4];
            else if (i < 4 + nb + nb + 1) v = poolofs[i - 4 - nb];
            h[i] = v;
        }
    }
}

// after the pack (stream order): publish the payload's size and the sequence number
__global__ void k_peer_signal(DsmPeerCtrl *ctrl, int rank, unsigned long long seq, const int32_t *nnew, const int32_t *poolofs, int nb, unsigned hb)
{
    long long n = 0;
    for (int i = 0; i < nb; i++) n += nnew[i];
    n += poolofs[nb];
    __threadfence_system();
    ctrl->bytes[rank] = (long long)hb + n * (long long)sizeof(dsm_surfel_t);
    __threadfence_system();
    st_release_sys(&ctrl->arrived[rank], seq);
}

extern "C" int dsm_comm_unique_id(void *id_out)
{
    if (!id_out) return DSM_E_INVALID;
    DsmNccl *api = nccl_api();
    if (!api) return DSM_E_NCCL;
    ncclUniqueId id;
    if (api->GetUniqueId(&id) != ncclSuccess) return DSM_E_NCCL;
    memcpy(id_out, &id, DSM_COMM_ID_BYTES);
    return DSM_OK;
}

extern "C" int dsm_comm_destroy(dsm_ctx *ctx)
{
    if (!ctx) return DSM_E_INVALID;
    DsmComm *c = ctx->comm;
    if (!c) return DSM_OK;
    cudaSetDevice(ctx->device);
    if (c->stream) cudaStreamSynchronize(c->stream);
    DsmNccl *api = nccl_api();
    if (c->comm && api) api->CommDestroy(c->comm);
    delete c; // unmaps the root's buffers, releases every buffer, stream and event
    ctx->comm = nullptr;
    return DSM_OK;
}

extern "C" int dsm_comm_init(dsm_ctx *ctx, const void *id, int rank, int nranks)
{
    if (!ctx || !id || nranks < 1 || rank < 0 || rank >= nranks) return DSM_E_INVALID;
    if (ctx->comm) return DSM_E_STATE;
    DsmNccl *api = nccl_api();
    if (!api)
    {
        snprintf(ctx->err, sizeof(ctx->err), "libnccl.so.2 could not be loaded: %s", dlerror());
        return DSM_E_NCCL;
    }
    CK(cudaSetDevice(ctx->device));
    DsmComm *c = new (std::nothrow) DsmComm();
    if (!c) return DSM_E_NOMEM;
    ctx->comm = c;
    c->rank = rank, c->nranks = nranks;
    {
        const char *e = getenv("DSM_GATHER_NCCL");
        c->force_nccl = (e && e[0] == '1') || nranks > DSM_MAX_RANKS;
    }
    ncclUniqueId uid;
    memcpy(&uid, id, DSM_COMM_ID_BYTES);
    NK(api->CommInitRank(&c->comm, nranks, uid, rank));
    c->own.stream(&c->stream);
    c->own.event(&c->ev_kernels);
    c->own.event(&c->ev_packed);
    c->pack_cap = payload_cap(ctx);
    c->own.device(&c->pack, c->pack_cap);
    c->own.device(&c->d_bytes, (size_t)nranks);
    c->own.host(&c->h_bytes, (size_t)nranks);
    c->own.host(&c->h_cnt, (size_t)ctx->p.max_batch);
    CK(c->own.take());
    c->ofs.assign((size_t)nranks + 1, 0);
    return DSM_OK;
}

// ---- peer-memory transport: host side ----
static void unmap_root(DsmComm *c)
{
    c->ipc_slots.reset();
    c->ipc_ctrl.reset();
    c->r_slots = nullptr, c->r_ctrl = nullptr;
}

// Collective over the communicator (every rank calls dsm_gather_deltas with the same root): maps the root's slots and
// control block into this process.  Leaves peer_ok false (-> NCCL transport) when any rank cannot map them.
static int peer_setup(dsm_ctx *ctx, int root)
{
    DsmComm *c = ctx->comm;
    DsmNccl *api = nccl_api();
    cudaStream_t cs = c->stream;
    CK(cudaStreamSynchronize(cs));
    unmap_root(c);
    c->peer_root = root, c->peer_ok = false, c->seq = 0;
    c->slot_bytes = (c->pack_cap + 255) / 256 * 256;
    if (!c->slots)
    {
        c->own.device(&c->slots, (size_t)c->nranks * c->slot_bytes);
        c->own.device(&c->ctrl, 1);
    }
    if (!c->poll)
    {
        c->own.stream(&c->poll);
        c->own.host(&c->h_arrived, DSM_MAX_RANKS);
    }
    CK(c->own.take());
    c->done_seq = 0;
    CK(cudaMemsetAsync(c->ctrl, 0, sizeof(DsmPeerCtrl), cs));
    CK(cudaStreamSynchronize(cs)); // zeroed before any peer can hold the handle
    if (c->nranks == 1)
    {
        c->r_slots = c->slots, c->r_ctrl = c->ctrl, c->peer_ok = true;
        return DSM_OK;
    }
    unsigned char mine[128];
    memset(mine, 0, sizeof(mine));
    cudaIpcMemHandle_t h_slots, h_ctrl;
    static_assert(sizeof(cudaIpcMemHandle_t) == 64, "handle size");
    bool good = cudaIpcGetMemHandle(&h_slots, c->slots) == cudaSuccess && cudaIpcGetMemHandle(&h_ctrl, c->ctrl) == cudaSuccess;
    cudaGetLastError();
    memcpy(mine, &h_slots, 64);
    memcpy(mine + 64, &h_ctrl, 64);
    if (!c->d_handles) c->own.device(&c->d_handles, (size_t)c->nranks * 128);
    CK(c->own.take());
    CK(cudaMemcpyAsync(c->d_handles + (size_t)c->rank * 128, mine, 128, cudaMemcpyHostToDevice, cs));
    NK(api->AllGather(c->d_handles + (size_t)c->rank * 128, c->d_handles, 128, ncclInt8, c->comm, cs));
    std::vector<unsigned char> all((size_t)c->nranks * 128);
    CK(cudaMemcpyAsync(all.data(), c->d_handles, all.size(), cudaMemcpyDeviceToHost, cs));
    CK(cudaStreamSynchronize(cs));
    if (c->rank == root)
        c->r_slots = c->slots, c->r_ctrl = c->ctrl;
    else if (good)
    {
        memcpy(&h_slots, all.data() + (size_t)root * 128, 64);
        memcpy(&h_ctrl, all.data() + (size_t)root * 128 + 64, 64);
        void *p = nullptr;
        if (cudaIpcOpenMemHandle(&p, h_slots, cudaIpcMemLazyEnablePeerAccess) == cudaSuccess) c->ipc_slots.reset(p);
        if (c->ipc_slots && cudaIpcOpenMemHandle(&p, h_ctrl, cudaIpcMemLazyEnablePeerAccess) == cudaSuccess) c->ipc_ctrl.reset(p);
        if (c->ipc_ctrl)
        {
            c->r_slots = static_cast<unsigned char *>(c->ipc_slots.get());
            c->r_ctrl = static_cast<DsmPeerCtrl *>(c->ipc_ctrl.get());
        }
        else
        {
            unmap_root(c);
            cudaGetLastError();
            good = false;
        }
    }
    // all ranks or none
    c->h_bytes[c->rank] = good ? 1 : 0;
    CK(cudaMemcpyAsync(c->d_bytes + c->rank, c->h_bytes + c->rank, sizeof(int64_t), cudaMemcpyHostToDevice, cs));
    NK(api->AllGather(c->d_bytes + c->rank, c->d_bytes, 1, ncclInt64, c->comm, cs));
    CK(cudaMemcpyAsync(c->h_bytes, c->d_bytes, (size_t)c->nranks * sizeof(int64_t), cudaMemcpyDeviceToHost, cs));
    CK(cudaStreamSynchronize(cs));
    bool all_good = true;
    for (int r = 0; r < c->nranks; r++) all_good &= c->h_bytes[r] == 1;
    if (!all_good && c->ipc_slots) unmap_root(c);
    c->peer_ok = all_good;
    return DSM_OK;
}

// Root: wait (on the host, polling the control block through a stream of its own) until every rank's payload of the last
// gather is complete, then fetch the sizes.  Other ranks: their own writes are done when the side stream is.
static int peer_wait(dsm_ctx *ctx)
{
    DsmComm *c = ctx->comm;
    CK(cudaStreamSynchronize(c->stream));
    if (!c->last_peer || c->rank != c->last_root || c->done_seq >= c->seq) return DSM_OK;
    for (int iter = 0;; iter++)
    {
        CK(cudaMemcpyAsync(c->h_arrived, c->ctrl->arrived, (size_t)c->nranks * sizeof(unsigned long long), cudaMemcpyDeviceToHost, c->poll));
        CK(cudaStreamSynchronize(c->poll));
        bool all = true;
        for (int r = 0; r < c->nranks; r++) all &= c->h_arrived[r] >= c->seq;
        if (all) break;
        if (iter > 400000)
        { // ~20 s
            snprintf(ctx->err, sizeof(ctx->err), "dsm_gather: a peer's payload did not arrive (sequence %llu)", c->seq);
            return DSM_E_NCCL;
        }
        if (iter > 100) usleep(50);
    }
    CK(cudaMemcpyAsync(c->h_bytes, c->ctrl->bytes, (size_t)c->nranks * sizeof(int64_t), cudaMemcpyDeviceToHost, c->poll));
    CK(cudaStreamSynchronize(c->poll));
    c->done_seq = c->seq;
    return DSM_OK;
}

// One gather over peer memory: nothing here waits on the host.
static int gather_peer(dsm_ctx *ctx, int root)
{
    DsmComm *c = ctx->comm;
    cudaStream_t cs = c->stream;
    const int nb = ctx->nb, S = ctx->d.S;
    const unsigned long long seq = ++c->seq;
    const unsigned hb = (unsigned)header_bytes(nb);
    CK(cudaEventRecord(c->ev_kernels, ctx->stream)); // the batch's kernels (all sub-batch streams are joined into it)
    CK(cudaStreamWaitEvent(cs, c->ev_kernels, 0));
    if (c->rank == root)
        k_peer_credit<<<1, 1, 0, cs>>>(c->ctrl, seq); // stream order: after the previous gather's completion on this stream
    else
        k_peer_wait_credit<<<1, 1, 0, cs>>>(c->r_ctrl, seq);
    unsigned char *slot = c->r_slots + (size_t)c->rank * c->slot_bytes;
    k_peer_pack<<<dim3(64, nb + 1), 256, 0, cs>>>(ctx->d.newsurf, ctx->d.nnew, ctx->d.pool, ctx->d.poolofs, S, nb, slot, hb);
    CK(cudaEventRecord(c->ev_packed, cs));
    CK(cudaStreamWaitEvent(ctx->stream, c->ev_packed, 0)); // later work on the compute stream may overwrite newsurf / pool
    k_peer_signal<<<1, 1, 0, cs>>>(c->r_ctrl, c->rank, seq, ctx->d.nnew, ctx->d.poolofs, nb, hb);
    if (c->rank == root) // completion is observed from the host (peer_wait): no kernel of the root ever spins on its peers
        for (int r = 0; r <= c->nranks; r++) c->ofs[r] = (size_t)r * c->slot_bytes;
    c->last_root = root;
    c->last_peer = true;
    CK(cudaGetLastError());
    return DSM_OK;
}

static int gather_nccl(dsm_ctx *ctx, int root);

extern "C" int dsm_gather_deltas(dsm_ctx *ctx, int root)
{
    if (!ctx) return DSM_E_INVALID;
    DsmComm *c = ctx->comm;
    DsmNccl *api = nccl_api();
    if (!c || !api) return DSM_E_STATE;
    if (root < 0 || root >= c->nranks) return DSM_E_INVALID;
    if (!ctx->ran || ctx->in_flight || ctx->res_active) return DSM_E_STATE; // the deltas of a dsm_batch_run batch
    CK(cudaSetDevice(ctx->device));
    if (!c->force_nccl && c->peer_root != root)
    {
        int rc = peer_setup(ctx, root);
        if (rc != DSM_OK) return rc;
    }
    return (!c->force_nccl && c->peer_ok) ? gather_peer(ctx, root) : gather_nccl(ctx, root);
}

static int gather_nccl(dsm_ctx *ctx, int root)
{
    DsmComm *c = ctx->comm;
    DsmNccl *api = nccl_api();
    const int nb = ctx->nb, S = ctx->d.S;
    // (1) new-surfel counts of the batch -> pinned memory (NCCL needs the payload's size on the host); this waits for the
    // batch's kernels
    CK(cudaStreamSynchronize(c->stream)); // the previous gather has consumed the staging buffers
    CK(cudaMemcpyAsync(c->h_cnt, ctx->d.nnew, (size_t)nb * sizeof(int32_t), cudaMemcpyDeviceToHost, ctx->stream));
    CK(cudaEventRecord(c->ev_kernels, ctx->stream));
    CK(cudaEventSynchronize(c->ev_kernels));
    size_t n_rec = (size_t)ctx->n_pool;
    for (int f = 0; f < nb; f++) n_rec += c->h_cnt[f];
    const unsigned hb = (unsigned)header_bytes(nb);
    const size_t my_bytes = hb + n_rec * sizeof(dsm_surfel_t);
    if (my_bytes > c->pack_cap) return DSM_E_CAPACITY;
    // (2) pack on the side stream: the payload a peer writes into its slot, here into the local send buffer
    cudaStream_t cs = c->stream;
    k_peer_pack<<<dim3(64, nb + 1), 256, 0, cs>>>(ctx->d.newsurf, ctx->d.nnew, ctx->d.pool, ctx->d.poolofs, S, nb, c->pack, hb);
    CK(cudaEventRecord(c->ev_packed, cs));
    CK(cudaStreamWaitEvent(ctx->stream, c->ev_packed, 0)); // later work on the compute stream may overwrite newsurf / pool
    // (3) byte counts of every rank
    c->h_bytes[c->rank] = (int64_t)my_bytes;
    CK(cudaMemcpyAsync(c->d_bytes + c->rank, c->h_bytes + c->rank, sizeof(int64_t), cudaMemcpyHostToDevice, cs));
    if (c->nranks > 1)
    {
        NK(api->AllGather(c->d_bytes + c->rank, c->d_bytes, 1, ncclInt64, c->comm, cs));
        CK(cudaMemcpyAsync(c->h_bytes, c->d_bytes, (size_t)c->nranks * sizeof(int64_t), cudaMemcpyDeviceToHost, cs));
        CK(cudaStreamSynchronize(cs));
    }
    // (4) payloads
    if (c->rank == root)
    {
        size_t total = 0;
        for (int r = 0; r < c->nranks; r++)
        {
            c->ofs[r] = total;
            total += ((size_t)c->h_bytes[r] + 255) / 256 * 256; // every payload starts 256-byte aligned
        }
        c->ofs[c->nranks] = total;
        if (total > c->recv_cap)
        { // grown on demand (first call: nranks payloads of this context's capacity)
            CK(cudaStreamSynchronize(cs));
            c->recv.reset();
            c->recv_cap = 0;
            size_t want = (size_t)c->nranks * ((c->pack_cap + 255) / 256 * 256);
            if (want < total) want = total;
            void *p = nullptr;
            CK(cudaMalloc(&p, want));
            c->recv.reset(static_cast<unsigned char *>(p));
            c->recv_cap = want;
        }
        CK(cudaMemcpyAsync(c->recv.get() + c->ofs[root], c->pack, my_bytes, cudaMemcpyDeviceToDevice, cs));
    }
    if (c->nranks > 1)
    {
        NK(api->GroupStart());
        if (c->rank == root)
        {
            for (int r = 0; r < c->nranks; r++)
                if (r != root) NK(api->Recv(c->recv.get() + c->ofs[r], (size_t)c->h_bytes[r], ncclInt8, r, c->comm, cs));
        }
        else
            NK(api->Send(c->pack, my_bytes, ncclInt8, root, c->comm, cs));
        NK(api->GroupEnd());
    }
    c->last_root = root;
    c->last_peer = false;
    CK(cudaGetLastError());
    return DSM_OK;
}

extern "C" int dsm_gather_wait(dsm_ctx *ctx)
{
    if (!ctx) return DSM_E_INVALID;
    if (!ctx->comm) return DSM_E_STATE;
    CK(cudaSetDevice(ctx->device));
    return peer_wait(ctx);
}

extern "C" int dsm_gathered_device(dsm_ctx *ctx, void **dev_ptr, size_t *rank_offsets)
{
    if (!ctx || !dev_ptr || !rank_offsets) return DSM_E_INVALID;
    DsmComm *c = ctx->comm;
    if (!c || c->last_root != c->rank) return DSM_E_STATE;
    *dev_ptr = c->last_peer ? c->slots : c->recv.get();
    for (int r = 0; r <= c->nranks; r++) rank_offsets[r] = c->ofs[r];
    return DSM_OK;
}

extern "C" int dsm_gathered_rank_bytes(dsm_ctx *ctx, int rank, size_t *bytes)
{
    if (!ctx || !bytes) return DSM_E_INVALID;
    DsmComm *c = ctx->comm;
    if (!c || c->last_root != c->rank) return DSM_E_STATE;
    if (rank < 0 || rank >= c->nranks) return DSM_E_INVALID;
    CK(cudaSetDevice(ctx->device));
    int rcw = peer_wait(ctx); // peer transport: the sizes arrive with the payloads
    if (rcw != DSM_OK) return rcw;
    *bytes = (size_t)c->h_bytes[rank];
    return DSM_OK;
}

extern "C" int dsm_gathered_download(dsm_ctx *ctx, int rank, void *host_out, size_t cap)
{
    if (!ctx || !host_out) return DSM_E_INVALID;
    DsmComm *c = ctx->comm;
    if (!c || c->last_root != c->rank) return DSM_E_STATE;
    if (rank < 0 || rank >= c->nranks) return DSM_E_INVALID;
    CK(cudaSetDevice(ctx->device));
    int rcw = peer_wait(ctx);
    if (rcw != DSM_OK) return rcw;
    const size_t nbytes = (size_t)c->h_bytes[rank];
    if (nbytes > cap) return DSM_E_CAPACITY;
    CK(cudaMemcpy(host_out, (c->last_peer ? c->slots : c->recv.get()) + c->ofs[rank], nbytes, cudaMemcpyDeviceToHost));
    return DSM_OK;
}
