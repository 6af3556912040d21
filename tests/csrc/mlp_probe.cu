// mlp_probe.cu -- one-block probes of the CUDA-core neural-ODE device functions (csrc/mlp.cuh), for
// tests/test_gpu_mlp_probe.py.  The production functions are called unchanged; this file only adds __global__ wrappers
// and extern "C" launchers over device pointers, for T = double (suffix _f64) and T = float (_f32).  Test-only: it is not
// part of libb200adj.so.
//
// Host arrays are the shared-memory images, row-major: X[64][32], y / L / F / JTL [2][32], H1 / H2 / D1 / D2 [64][32].
// Every launcher runs one block of MLP_THREADS threads (mlp_reduce_kernel: its production launch), waits for it and
// returns the cudaError_t (0 = success).
#include "mlp.cuh"

using namespace b200adj;

namespace {

template <class T>
__device__ void load(T (*dst)[MLP_TB], int rows, const T* src) {
    for (int x = threadIdx.x; x < rows * MLP_TB; x += MLP_THREADS) dst[x / MLP_TB][x % MLP_TB] = src[x];
}
template <class T>
__device__ void store(const T (*src)[MLP_TB], int rows, T* dst) {
    for (int x = threadIdx.x; x < rows * MLP_TB; x += MLP_THREADS) dst[x] = src[x / MLP_TB][x % MLP_TB];
}

// out[m][b] = sum_k Wk[k][m] X[k][b] with Wk = W2F (transposed = 0: W2 X) or W2B (transposed = 1: W2' X)
template <class T>
__global__ void __launch_bounds__(MLP_THREADS) gemm_probe(const T* p, const T* X, int transposed, T* out) {
    extern __shared__ __align__(16) unsigned char probe_smem[];
    MlpSmem<T>& s = *reinterpret_cast<MlpSmem<T>*>(probe_smem);
    mlp_load_params<T>(s, p);
    load<T>(s.H1, MLP_H, X);
    __syncthreads();
    const int m0 = (threadIdx.x / 16) * 4, b0 = (threadIdx.x % 16) * 2;
    T acc[4][2];
    mlp_gemm<T>(transposed ? s.W2B : s.W2F, s.H1, m0, b0, acc);
    for (int r = 0; r < 4; r++) { out[(m0 + r) * MLP_TB + b0] = acc[r][0]; out[(m0 + r) * MLP_TB + b0 + 1] = acc[r][1]; }
}

// mlp_forward at y, then mlp_backward of L: F, H1, H2, D2, D1, JTL
template <class T>
__global__ void __launch_bounds__(MLP_THREADS) layers_probe(const T* p, const T* y, const T* L, T* F, T* H1, T* H2, T* D2, T* D1, T* JTL) {
    extern __shared__ __align__(16) unsigned char probe_smem[];
    MlpSmem<T>& s = *reinterpret_cast<MlpSmem<T>*>(probe_smem);
    mlp_load_params<T>(s, p);
    load<T>(s.y, MLP_D, y);
    load<T>(s.L, MLP_D, L);
    __syncthreads();
    mlp_forward<T>(s);
    mlp_backward<T>(s);
    store<T>(s.F, MLP_D, F); store<T>(s.H1, MLP_H, H1); store<T>(s.H2, MLP_H, H2);
    store<T>(s.D2, MLP_H, D2); store<T>(s.D1, MLP_H, D1); store<T>(s.JTL, MLP_D, JTL);
}

// mlp_accumulate(c, nvalid) over the given activations, then mlp_store_grad into out[P]
template <class T>
__global__ void __launch_bounds__(MLP_THREADS) accumulate_probe(const T* y, const T* L, const T* H1, const T* H2, const T* D1, const T* D2,
                                                                T c, int nvalid, T* out) {
    extern __shared__ __align__(16) unsigned char probe_smem[];
    MlpSmem<T>& s = *reinterpret_cast<MlpSmem<T>*>(probe_smem);
    load<T>(s.y, MLP_D, y); load<T>(s.L, MLP_D, L);
    load<T>(s.H1, MLP_H, H1); load<T>(s.H2, MLP_H, H2); load<T>(s.D1, MLP_H, D1); load<T>(s.D2, MLP_H, D2);
    __syncthreads();
    MlpGrad<T> g;
    for (int r = 0; r < 4; r++)
        for (int q = 0; q < 4; q++) g.w2[r][q] = 0;
    g.a = g.b = g.c = g.d = 0;
    mlp_accumulate<T>(s, g, c, nvalid);
    mlp_store_grad<T>(g, out);
}

template <class K, class... A>
int launch(int smem, K kernel, A... args) {
    cudaError_t e = cudaFuncSetAttribute(kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, smem);
    if (e != cudaSuccess) return (int)e;
    kernel<<<1, MLP_THREADS, smem>>>(args...);
    e = cudaGetLastError();
    if (e != cudaSuccess) return (int)e;
    return (int)cudaDeviceSynchronize();
}

template <class T>
int reduce(const T* partials, T* dp, int nblocks) {
    mlp_reduce_kernel<T><<<(MLP_P + 255) / 256, 256>>>(partials, dp, nblocks);
    cudaError_t e = cudaGetLastError();
    if (e != cudaSuccess) return (int)e;
    return (int)cudaDeviceSynchronize();
}

}  // namespace

#define B200_MLP_PROBES(T, SFX)                                                                                              \
    extern "C" int probe_gemm_##SFX(const T* p, const T* X, int transposed, T* out) {                                        \
        return launch((int)sizeof(MlpSmem<T>), gemm_probe<T>, p, X, transposed, out);                                       \
    }                                                                                                                        \
    extern "C" int probe_layers_##SFX(const T* p, const T* y, const T* L, T* F, T* H1, T* H2, T* D2, T* D1, T* JTL) {         \
        return launch((int)sizeof(MlpSmem<T>), layers_probe<T>, p, y, L, F, H1, H2, D2, D1, JTL);                            \
    }                                                                                                                        \
    extern "C" int probe_accumulate_##SFX(const T* y, const T* L, const T* H1, const T* H2, const T* D1, const T* D2, T c,   \
                                          int nvalid, T* out) {                                                              \
        return launch((int)sizeof(MlpSmem<T>), accumulate_probe<T>, y, L, H1, H2, D1, D2, c, nvalid, out);                   \
    }                                                                                                                        \
    extern "C" int probe_reduce_##SFX(const T* partials, T* dp, int nblocks) { return reduce<T>(partials, dp, nblocks); }
B200_MLP_PROBES(double, f64)
B200_MLP_PROBES(float, f32)
#undef B200_MLP_PROBES
