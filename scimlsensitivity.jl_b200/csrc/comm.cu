// comm.cu -- multi-GPU behind the C ABI (SURVEY.md 8b/8e): one handle per GPU (one process per GPU, or several handles
// in one process), ensemble members sharded over the handles, and exactly ONE collective per gradient -- the sum of
// dG/dp over the ranks when the parameters are shared -- issued by b200adj_reverse itself on the handle's stream.
//
// NCCL is bound at run time with dlopen("libnccl.so.2") (the copy a host process already carries -- PyTorch's bundled
// one, or the system library for a Julia host), so libb200adj.so has no link-time dependency on it and single-GPU users
// never load it.  The unique id travels through the host's own channel (MPI / Distributed.jl / torch.distributed store):
//   rank 0: b200adj_comm_unique_id(id)  ->  broadcast the 128 bytes  ->  every rank: b200adj_comm_init(h, nranks, rank, id).
#include <dlfcn.h>

#include "handle.h"

using namespace b200adj;

namespace {

typedef struct { char internal[128]; } nccl_uid;
typedef void* nccl_comm_t;
enum { NCCL_FLOAT32 = 7, NCCL_FLOAT64 = 8, NCCL_SUM = 0 };

struct Nccl {
    void* lib = nullptr;
    int (*GetUniqueId)(nccl_uid*) = nullptr;
    int (*CommInitRank)(nccl_comm_t*, int, nccl_uid, int) = nullptr;
    int (*AllReduce)(const void*, void*, size_t, int, int, nccl_comm_t, cudaStream_t) = nullptr;
    int (*AllGather)(const void*, void*, size_t, int, nccl_comm_t, cudaStream_t) = nullptr;
    int (*CommDestroy)(nccl_comm_t) = nullptr;
    int (*GroupStart)() = nullptr;
    int (*GroupEnd)() = nullptr;
    const char* (*GetErrorString)(int) = nullptr;
    std::string err;
};

// loaded once per process; immutable afterwards (the "no global state" rule of the ABI is about mutable solver state)
Nccl* nccl() {
    static Nccl n;
    static bool tried = false;
    if (!tried) {
        tried = true;
        const char* names[] = {"libnccl.so.2", "libnccl.so"};
        for (const char* nm : names) { n.lib = dlopen(nm, RTLD_NOW | RTLD_GLOBAL); if (n.lib) break; }
        if (!n.lib) { const char* e = dlerror(); n.err = std::string("dlopen(libnccl.so.2) failed: ") + (e ? e : "?"); return &n; }
        n.GetUniqueId = (int (*)(nccl_uid*))dlsym(n.lib, "ncclGetUniqueId");
        n.CommInitRank = (int (*)(nccl_comm_t*, int, nccl_uid, int))dlsym(n.lib, "ncclCommInitRank");
        n.AllReduce = (int (*)(const void*, void*, size_t, int, int, nccl_comm_t, cudaStream_t))dlsym(n.lib, "ncclAllReduce");
        n.AllGather = (int (*)(const void*, void*, size_t, int, nccl_comm_t, cudaStream_t))dlsym(n.lib, "ncclAllGather");
        n.CommDestroy = (int (*)(nccl_comm_t))dlsym(n.lib, "ncclCommDestroy");
        n.GetErrorString = (const char* (*)(int))dlsym(n.lib, "ncclGetErrorString");
        n.GroupStart = (int (*)())dlsym(n.lib, "ncclGroupStart");
        n.GroupEnd = (int (*)())dlsym(n.lib, "ncclGroupEnd");
        if (!n.GetUniqueId || !n.CommInitRank || !n.AllReduce || !n.CommDestroy) { n.err = "libnccl: missing symbols"; n.lib = nullptr; }
    }
    return &n;
}

}  // namespace

namespace b200adj {

// sum `count` reals (the handle's ABI element type) over the ranks, in place, on the handle's stream
bool comm_fused_ready(const Handle* h) { return h->p2p.nranks > 1; }

int comm_allreduce(Handle* h, void* buf, size_t count) {
    if (!h->nccl_comm || h->nranks <= 1) return B200ADJ_OK;
    Nccl* n = nccl();
    const int dt = esz(h->cfg) == sizeof(double) ? NCCL_FLOAT64 : NCCL_FLOAT32;
    const int rc = n->AllReduce(buf, buf, count, dt, NCCL_SUM, (nccl_comm_t)h->nccl_comm, h->stream);
    if (rc != 0) { h->err = std::string("ncclAllReduce: ") + (n->GetErrorString ? n->GetErrorString(rc) : "error"); return B200ADJ_ERR_CUDA; }
    h->launches++;
    return B200ADJ_OK;
}

// ---- mailboxes of the fused all-reduce ----
constexpr size_t P2P_SLOT_DOUBLES = 2 * (size_t)P2P_MAXRANKS * P2P_PMAX;                       // two parities
constexpr size_t P2P_MAILBOX_BYTES = P2P_SLOT_DOUBLES * sizeof(double) + P2P_MAXRANKS * sizeof(unsigned long long);
static void p2p_point(P2PComm* pc, int r, void* base) {
    pc->slots[r] = (double*)base;
    pc->flags[r] = (unsigned long long*)((char*)base + P2P_SLOT_DOUBLES * sizeof(double));
}
static void p2p_release(Handle* h) {
    for (int r = 0; r < P2P_MAXRANKS; r++) if (h->p2p_ipc_open[r]) { cudaIpcCloseMemHandle(h->p2p_ipc_open[r]); h->p2p_ipc_open[r] = nullptr; }
    dev_free(h, h->p2p_mailbox);
    memset(&h->p2p, 0, sizeof(h->p2p)); h->p2p_epoch = 0;
}
static bool p2p_alloc(Handle* h) {
    if (cudaSetDevice(h->cfg.device) != cudaSuccess) return false;
    if (dev_malloc(h, &h->p2p_mailbox, P2P_MAILBOX_BYTES) != cudaSuccess) { cudaGetLastError(); h->p2p_mailbox = nullptr; return false; }
    return cudaMemset(h->p2p_mailbox, 0, P2P_MAILBOX_BYTES) == cudaSuccess && cudaDeviceSynchronize() == cudaSuccess;
}
// one process per GPU: exchange CUDA IPC handles of the mailboxes through the communicator itself (one ncclAllGather)
static void p2p_setup_multiprocess(Handle* h) {
    Nccl* n = nccl();
    if (!n->AllGather || h->nranks > P2P_MAXRANKS || h->cfg.P > P2P_PMAX) return;
    if (!p2p_alloc(h)) { p2p_release(h); return; }
    cudaIpcMemHandle_t mine, all[P2P_MAXRANKS];
    void *d_send = nullptr, *d_recv = nullptr;
    bool ok = cudaIpcGetMemHandle(&mine, h->p2p_mailbox) == cudaSuccess &&
              cudaMalloc(&d_send, sizeof(mine)) == cudaSuccess && cudaMalloc(&d_recv, sizeof(mine) * h->nranks) == cudaSuccess &&
              cudaMemcpy(d_send, &mine, sizeof(mine), cudaMemcpyHostToDevice) == cudaSuccess;
    // every rank must take part in the collective even if its own preparation failed: a failed rank sends zeros
    if (!ok && d_send) cudaMemset(d_send, 0, sizeof(mine));
    if (d_send && d_recv && n->AllGather(d_send, d_recv, sizeof(mine), 0 /* ncclChar */, (nccl_comm_t)h->nccl_comm, h->stream) == 0 &&
        cudaStreamSynchronize(h->stream) == cudaSuccess && cudaMemcpy(all, d_recv, sizeof(mine) * h->nranks, cudaMemcpyDeviceToHost) == cudaSuccess) {
        P2PComm pc; memset(&pc, 0, sizeof(pc));
        for (int r = 0; r < h->nranks && ok; r++) {
            if (r == h->rank) { p2p_point(&pc, r, h->p2p_mailbox); continue; }
            bool zero = true;
            for (size_t b = 0; b < sizeof(mine); b++) zero = zero && ((const char*)&all[r])[b] == 0;
            void* ptr = nullptr;
            if (zero || cudaIpcOpenMemHandle(&ptr, all[r], cudaIpcMemLazyEnablePeerAccess) != cudaSuccess) { cudaGetLastError(); ok = false; break; }
            h->p2p_ipc_open[r] = ptr;
            p2p_point(&pc, r, ptr);
        }
        if (ok) { pc.nranks = h->nranks; pc.rank = h->rank; h->p2p = pc; }
    } else ok = false;
    cudaFree(d_send); cudaFree(d_recv);
    // all ranks must agree on the path: a second tiny collective carries the verdict (sum of failures)
    double verdict = ok ? 0.0 : 1.0, *d_v = nullptr;
    if (cudaMalloc(&d_v, sizeof(double)) == cudaSuccess) {
        cudaMemcpy(d_v, &verdict, sizeof(double), cudaMemcpyHostToDevice);
        if (n->AllReduce(d_v, d_v, 1, NCCL_FLOAT64, NCCL_SUM, (nccl_comm_t)h->nccl_comm, h->stream) == 0 && cudaStreamSynchronize(h->stream) == cudaSuccess)
            cudaMemcpy(&verdict, d_v, sizeof(double), cudaMemcpyDeviceToHost);
        else verdict = 1.0;
        cudaFree(d_v);
    } else verdict = 1.0;
    if (verdict != 0.0) p2p_release(h);
}

void comm_release(Handle* h) {
    p2p_release(h);
    if (h->nccl_comm) { Nccl* n = nccl(); if (n->lib) n->CommDestroy((nccl_comm_t)h->nccl_comm); h->nccl_comm = nullptr; }
    h->nranks = 1; h->rank = 0;
}

}  // namespace b200adj

extern "C" {

int32_t b200adj_comm_unique_id(void* id_out) {
    if (!id_out) return B200ADJ_ERR_INVALID;
    Nccl* n = nccl();
    if (!n->lib) return B200ADJ_ERR_UNSUPPORTED;
    nccl_uid id;
    if (n->GetUniqueId(&id) != 0) return B200ADJ_ERR_CUDA;
    memcpy(id_out, &id, sizeof(id));
    return B200ADJ_OK;
}

int32_t b200adj_comm_init(void* handle, int32_t nranks, int32_t rank, const void* unique_id) {
    if (!handle) return B200ADJ_ERR_INVALID;
    Handle* h = (Handle*)handle;
    if (nranks < 1 || rank < 0 || rank >= nranks || (nranks > 1 && !unique_id)) { h->err = "comm_init: bad nranks/rank/id"; return B200ADJ_ERR_INVALID; }
    comm_release(h);
    if (nranks == 1) return B200ADJ_OK;
    Nccl* n = nccl();
    if (!n->lib) { h->err = n->err; return B200ADJ_ERR_UNSUPPORTED; }
    CUDA_TRY(h, cudaSetDevice(h->cfg.device));
    nccl_uid id;
    memcpy(&id, unique_id, sizeof(id));
    nccl_comm_t comm = nullptr;
    const int rc = n->CommInitRank(&comm, nranks, id, rank);
    if (rc != 0) { h->err = std::string("ncclCommInitRank: ") + (n->GetErrorString ? n->GetErrorString(rc) : "error"); return B200ADJ_ERR_CUDA; }
    h->nccl_comm = comm; h->nranks = nranks; h->rank = rank;
    p2p_setup_multiprocess(h);            // mailboxes of the fused all-reduce (falls back to ncclAllReduce when P2P is unavailable)
    return B200ADJ_OK;
}

int32_t b200adj_comm_init_all(void** handles, int32_t n) {
    // single-process hosts (one Julia / Python process driving all GPUs of the box): the n handles become ranks 0..n-1 of one
    // communicator; the ncclCommInitRank calls are grouped so that one thread can issue them
    if (!handles || n < 1) return B200ADJ_ERR_INVALID;
    for (int i = 0; i < n; i++) if (!handles[i]) return B200ADJ_ERR_INVALID;
    if (n == 1) { comm_release((Handle*)handles[0]); return B200ADJ_OK; }
    Nccl* nc = nccl();
    Handle* h0 = (Handle*)handles[0];
    if (!nc->lib || !nc->GroupStart || !nc->GroupEnd) { h0->err = nc->err.empty() ? "libnccl: ncclGroupStart missing" : nc->err; return B200ADJ_ERR_UNSUPPORTED; }
    nccl_uid id;
    if (nc->GetUniqueId(&id) != 0) { h0->err = "ncclGetUniqueId failed"; return B200ADJ_ERR_CUDA; }
    std::vector<nccl_comm_t> comms((size_t)n, nullptr);
    for (int i = 0; i < n; i++) comm_release((Handle*)handles[i]);
    int rc = nc->GroupStart();
    for (int i = 0; i < n && rc == 0; i++) {
        Handle* h = (Handle*)handles[i];
        if (cudaSetDevice(h->cfg.device) != cudaSuccess) { rc = -1; break; }
        rc = nc->CommInitRank(&comms[i], n, id, i);
    }
    const int rc2 = nc->GroupEnd();
    if (rc != 0 || rc2 != 0) { h0->err = std::string("ncclCommInitRank (grouped): ") + (nc->GetErrorString ? nc->GetErrorString(rc ? rc : rc2) : "error"); return B200ADJ_ERR_CUDA; }
    for (int i = 0; i < n; i++) { Handle* h = (Handle*)handles[i]; h->nccl_comm = comms[i]; h->nranks = n; h->rank = i; }
    // mailboxes of the fused all-reduce: one process => plain peer access between the devices
    bool ok = n <= P2P_MAXRANKS;
    for (int i = 0; i < n && ok; i++) ok = ((Handle*)handles[i])->cfg.P <= P2P_PMAX && p2p_alloc((Handle*)handles[i]);
    for (int i = 0; i < n && ok; i++)
        for (int j = 0; j < n && ok; j++) {
            const int di = ((Handle*)handles[i])->cfg.device, dj = ((Handle*)handles[j])->cfg.device;
            if (di == dj) continue;
            int can = 0;
            if (cudaDeviceCanAccessPeer(&can, di, dj) != cudaSuccess || !can) { ok = false; break; }
            cudaSetDevice(di);
            const cudaError_t e = cudaDeviceEnablePeerAccess(dj, 0);
            if (e != cudaSuccess && e != cudaErrorPeerAccessAlreadyEnabled) ok = false;
            cudaGetLastError();
        }
    for (int i = 0; i < n; i++) {
        Handle* h = (Handle*)handles[i];
        if (!ok) { p2p_release(h); continue; }
        P2PComm pc; memset(&pc, 0, sizeof(pc));
        for (int r = 0; r < n; r++) p2p_point(&pc, r, ((Handle*)handles[r])->p2p_mailbox);
        pc.nranks = n; pc.rank = i; h->p2p = pc;
    }
    return B200ADJ_OK;
}

int32_t b200adj_comm_allreduce(void* handle, void* buf, int64_t count) {
    if (!handle || !buf || count < 0) return B200ADJ_ERR_INVALID;
    Handle* h = (Handle*)handle;
    if (h->nranks <= 1) return B200ADJ_OK;
    if (!h->cfg.buffers_on_device) { h->err = "comm_allreduce: device buffers only (host results are reduced inside b200adj_reverse)"; return B200ADJ_ERR_INVALID; }
    CUDA_TRY(h, cudaSetDevice(h->cfg.device));
    return comm_allreduce(h, buf, (size_t)count);
}

int32_t b200adj_comm_is_fused(void* handle) {
    return (handle && comm_fused_ready((Handle*)handle) && !(((Handle*)handle)->cfg.flags & B200ADJ_FLAG_NCCL_ALLREDUCE)) ? 1 : 0;
}

int32_t b200adj_comm_size(void* handle, int32_t* nranks, int32_t* rank) {
    if (!handle) return B200ADJ_ERR_INVALID;
    Handle* h = (Handle*)handle;
    if (nranks) *nranks = h->nranks;
    if (rank) *rank = h->rank;
    return B200ADJ_OK;
}

}  // extern "C"
