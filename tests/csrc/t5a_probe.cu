// t5a_probe.cu -- probes of the adaptive Tsit5 framework (csrc/tsit5_adaptive.cuh) for tests/test_gpu_t5a_probe.py: the
// reverse pass's lookup T5Dense<D>::eval on test-supplied records, and a copy of the dense solutions a handle's forward and
// QuadratureAdjoint reverse passes stored.  The production functions are called unchanged; this file only adds a
// __global__ wrapper and extern "C" entry points.  Test-only: it is not part of libb200adj.so.  Entry points wait for
// their work and return the cudaError_t (0 = success).
#include "handle.h"

using namespace b200adj;

namespace {

// ---- T5Dense<D>::eval: one member per thread walks its query sequence, as the reverse solve does ----
// records member-major recs[N][stride][8 D + 4], knots[N][stride], nk[N] intervals per member; queries tq[N][Q], right[N][Q];
// out y[N][Q][D], iv[N][Q] (the interval the lookup holds after the query), buf[N][Q] (the record buffer it reads).
// Shared memory is carved as t5a_reverse_kernel carves it: [2][blockDim.x][t5_pitch] record buffers, then [blockDim.x]
// mbarriers.
template <int D>
__global__ void t5_dense_kernel(const __grid_constant__ T5aArgs a, const double* recs, const double* knots, const int* nk, int stride,
                                int64_t N, int Q, const double* tq, const int* right, double* y, int* iv, int* buf) {
    constexpr int REC = t5_rec<D>();
    extern __shared__ __align__(16) double s_t5_dense[];
    const int bufstride = (int)blockDim.x * t5_pitch<D>();
    uint64_t* my_bar = reinterpret_cast<uint64_t*>(s_t5_dense + (size_t)2 * bufstride) + threadIdx.x;
    const int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= N) return;
    mbar_init(my_bar, 1);
    mbar_fence_init();
    T5Dense<D> sol{a, recs + i * stride * REC, knots + i * stride, nk[i], s_t5_dense + (size_t)threadIdx.x * t5_pitch<D>(), bufstride, my_bar};
    sol.cur = sol.n - 1;
    for (int k = 0; k < Q; k++) {
        const int64_t o = i * Q + k;
        sol.eval(tq[o], right[o] != 0, y + o * D);
        iv[o] = sol.civ;
        buf[o] = sol.cb;
    }
    if (sol.aiv >= 0) sol.arrived();      // the record of the interval below is still on its way: no bulk copy outlives the CTA
}

template <int D>
int run_dense(int block, const double* recs, const double* knots, const int* nk, int stride, long long N, int Q, const double* tq,
              const int* right, double* y, int* iv, int* buf) {
    T5aArgs a;
    memset(&a, 0, sizeof(a));
    const size_t smem = (size_t)block * (2 * t5_pitch<D>() * sizeof(double) + sizeof(uint64_t));
    cudaFuncSetAttribute(t5_dense_kernel<D>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem);
    t5_dense_kernel<D><<<(unsigned)((N + block - 1) / block), block, smem>>>(a, recs, knots, nk, stride, N, Q, tq, right, y, iv, buf);
    const cudaError_t e = cudaGetLastError();
    if (e != cudaSuccess) return (int)e;
    return (int)cudaDeviceSynchronize();
}

}  // namespace

extern "C" {

int probe_t5_dense(int D, int block, const double* recs, const double* knots, const int* nk, int stride, long long N, int Q,
                   const double* tq, const int* right, double* y, int* iv, int* buf) {
    switch (D) {
        case 1: return run_dense<1>(block, recs, knots, nk, stride, N, Q, tq, right, y, iv, buf);
        case 2: return run_dense<2>(block, recs, knots, nk, stride, N, Q, tq, right, y, iv, buf);
        case 3: return run_dense<3>(block, recs, knots, nk, stride, N, Q, tq, right, y, iv, buf);
        default: return (int)cudaErrorInvalidValue;
    }
}

// The dense solutions of an adaptive Tsit5 handle (an opaque b200adj handle, after b200adj_forward), copied to host buffers:
// knots ftT[N][maxs + 1], records frecT[N][maxs + 1][8 d + 4], fn[N]; after a QuadratureAdjoint reverse pass also the
// reverse records rrec[N][maxs][quad_pad(3 + 8 d)] = (t, h, z[d], k[7][d], 1/h), rend[N][maxs] = t + h and rn[N] (null
// pointers: not copied).  *maxs and *rwp are set first; a call with ftT null only reports them.
int probe_t5a_records(void* handle, int* maxs, int* rwp, double* ftT, double* frecT, int* fn, double* rrec, double* rend, int* rn) {
    Handle* h = static_cast<Handle*>(handle);
    if (!h || h->path != Path::T5A) return (int)cudaErrorInvalidValue;
    const size_t N = (size_t)h->cfg.N, MS = (size_t)h->maxs, d = (size_t)h->cfg.d;
    *maxs = h->maxs;
    *rwp = quad_pad(3 + 8 * (int)d);
    if (!ftT) return 0;
    cudaError_t e = cudaDeviceSynchronize();
    if (e != cudaSuccess) return (int)e;
    auto get = [&](void* dst, const void* src, size_t bytes) {
        if (e == cudaSuccess && dst) e = src ? cudaMemcpy(dst, src, bytes, cudaMemcpyDeviceToHost) : cudaErrorInvalidValue;
    };
    get(ftT, h->r_ftT, N * (MS + 1) * sizeof(double));
    get(frecT, h->r_frecT, N * (MS + 1) * (8 * d + 4) * sizeof(double));
    get(fn, h->r_fn, N * sizeof(int32_t));
    get(rrec, h->r_rrec, N * MS * (size_t)*rwp * sizeof(double));
    get(rend, h->r_rend, N * MS * sizeof(double));
    get(rn, h->r_rn, N * sizeof(int32_t));
    return (int)e;
}

}  // extern "C"
