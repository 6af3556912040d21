// fixed_probe.cu -- a copy of what the fixed-step Tsit5 kernels (csrc/ode_tsit5.cuh) stored in a handle, for
// tests/test_gpu_fixed_probe.py: the forward checkpoints and, after a QuadratureAdjoint reverse pass, its dense reverse
// solution.  Nothing here launches a kernel.  Test-only: it is not part of libb200adj.so.  The entry point waits for its
// copies and returns the cudaError_t (0 = success).
#include "handle.h"

using namespace b200adj;

extern "C" {

// The buffers of a fixed-step Tsit5 handle (an opaque b200adj handle, after b200adj_forward), copied to host buffers:
// ckpt[rows][d][Npad] (rows = S + 1, or ceil(S / C) + 1 under checkpoint_every = C > 1; row m holds u_{mC}, the last row
// u_S) and, after a QuadratureAdjoint reverse pass, adj[S][8][d][Npad] (lambda(t_{n+1}) after the jump there, then
// ka'[0..6] of reverse step n).  Elements are the handle's real type (esz = 8, or 4 for an F32 handle).  *S, *rows,
// *ckpt_every, *Npad and *esz are set first; a call with ckpt null only reports them; adj null: not copied.
int probe_fixed_buffers(void* handle, int* S, int* rows, int* ckpt_every, long long* Npad, int* esz_out, void* ckpt, void* adj) {
    Handle* h = static_cast<Handle*>(handle);
    if (!h || h->path != Path::FIXED || !h->d_ckpt) return (int)cudaErrorInvalidValue;
    const int C = h->ckpt_every;
    const size_t d = (size_t)h->cfg.d, e = esz(h->cfg), np = (size_t)h->Npad;
    *S = h->S;
    *rows = C > 1 ? (h->S + C - 1) / C + 1 : h->S + 1;
    *ckpt_every = C;
    *Npad = (long long)h->Npad;
    *esz_out = (int)e;
    if (!ckpt) return 0;
    cudaError_t r = cudaStreamSynchronize(h->stream);
    if (r == cudaSuccess) r = cudaMemcpy(ckpt, h->d_ckpt, (size_t)*rows * d * np * e, cudaMemcpyDeviceToHost);
    if (r == cudaSuccess && adj)
        r = h->d_adj_dense ? cudaMemcpy(adj, h->d_adj_dense, (size_t)h->S * 8 * d * np * e, cudaMemcpyDeviceToHost) : cudaErrorInvalidValue;
    return (int)r;
}

}  // extern "C"
