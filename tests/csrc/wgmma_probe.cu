// wgmma_probe.cu -- one-CTA probes of the tensor-core building blocks of the bf16 neural-ODE kernels (csrc/wgmma.cuh,
// csrc/mlp_tc.cuh, csrc/mlp_tc_wide.cuh), for tests/test_gpu_wgmma_probe.py.  The production device functions are called
// unchanged; this file only adds __global__ wrappers and extern "C" launchers over device pointers.  Test-only: it is not
// part of libb200adj.so.
//
// Host arrays are row-major fp32: a tile of F features is [rows][F], member inputs are [member][2].  Every launcher runs one
// CTA of 128 threads, waits for it and returns the cudaError_t of the launch (0 = success).
#include "mlp_tc_wide.cuh"

using namespace b200adj;

namespace {

// rows [0, rows) of a K-major tile of F features from src[rows][F] (values meant to be exact in bf16)
template <int F>
__device__ void fill_tile(unsigned char* tile, int rows, const float* src) {
    for (int x = threadIdx.x; x < rows * (F / 8); x += blockDim.x) {
        const float* v = src + (x / (F / 8)) * F + 8 * (x % (F / 8));
        *tc_chunk<F>(tile, x / (F / 8), x % (F / 8)) =
            make_uint4(pack_bf16(v[0], v[1]), pack_bf16(v[2], v[3]), pack_bf16(v[4], v[5]), pack_bf16(v[6], v[7]));
    }
}
// generic-proxy tile stores made visible to the wgmma (async) proxy of every thread
__device__ void tiles_ready() {
    asm volatile("fence.proxy.async.shared::cta;" ::: "memory");
    __syncthreads();
}
__device__ void copy_D(const float* D, int rows, float* out) {
    for (int x = threadIdx.x; x < rows * 64; x += blockDim.x) out[x] = D[(x / 64) * TC_DP + x % 64];
}

// ---- member GEMM: D = (rows of tile, features 0..63) . B', B = W2 (w2t = 0) or W2T (w2t = 1), tile = TB (F = 80) / TA (F = 128)
template <int F>
__global__ void __launch_bounds__(TC_M) tc_member_probe(const float* p, const float* a, int w2t, float* D) {
    extern __shared__ __align__(128) unsigned char probe_smem[];
    TcSmem& s = *reinterpret_cast<TcSmem*>(probe_smem);
    tc_setup(s, p);
    unsigned char* tile = F == TC_TB_F ? s.TB : s.TA;
    fill_tile<F>(tile, TC_ROWS, a);                       // all 64 MMA rows, the 32 pad rows included
    tiles_ready();
    float d[32];
    tc_member_mma(d, smem_u32(tile), (F / 8) * 128, smem_u32(w2t ? s.W2T : s.W2));
    if (threadIdx.x < 64) tc_stage(s.D, d, 0);            // accumulator rows 0..31 = the members
    __syncthreads();
    copy_D(s.D, TC_MEM, D);
}
template <int F>
__global__ void __launch_bounds__(TCW_M) tcw_member_probe(const float* p, const float* a, int w2t, float* D) {
    extern __shared__ __align__(128) unsigned char probe_smem[];
    TcwSmem& s = *reinterpret_cast<TcwSmem*>(probe_smem);
    tcw_setup(s, p);
    unsigned char* tile = F == TC_TB_F ? s.TB : s.TA;
    fill_tile<F>(tile, TCW_M, a);
    tiles_ready();
    tcw_member_mma(s, tile, (F / 8) * 128, w2t ? s.W2T : s.W2);
    __syncthreads();
    copy_D(s.D, TCW_M, D);
}

// ---- gradient GEMM: R rounds of G1 += TA' TB, G2 += TH' TC with new tile contents per round, then the parameter store.
// Round r reads ta + r * RAB * 128, tb + r * RAB * 80, th + r * RHC * 128, tc + r * RHC * 16.
template <class S, int RAB, int RHC, int KS>
__device__ void grad_rounds(S& s, int R, const float* ta, const float* tb, const float* th, const float* tc, float* out) {
    TcGrad g;
    g.zero();
#pragma unroll 1
    for (int r = 0; r < R; r++) {
        fill_tile<TC_TA_F>(s.TA, RAB, ta + r * RAB * TC_TA_F);
        fill_tile<TC_TB_F>(s.TB, RAB, tb + r * RAB * TC_TB_F);
        fill_tile<TC_TA_F>(s.TH, RHC, th + r * RHC * TC_TA_F);
        fill_tile<TC_TC_F>(s.TC, RHC, tc + r * RHC * TC_TC_F);
        tiles_ready();
        tc_grad_mma<KS>(g, smem_u32(s.TA), smem_u32(s.TB), smem_u32(s.TH), smem_u32(s.TC));
        wgmma_wait_all();                                 // the kernels' discipline: every warp's wait, then a barrier,
        __syncthreads();                                  // before any tile is rewritten
    }
    tc_grad_store(g, out);
}
__global__ void __launch_bounds__(TC_M) tc_grad_probe(const float* p, int R, const float* ta, const float* tb, const float* th, const float* tc, float* out) {
    extern __shared__ __align__(128) unsigned char probe_smem[];
    TcSmem& s = *reinterpret_cast<TcSmem*>(probe_smem);
    tc_setup(s, p);
    grad_rounds<TcSmem, TC_ROWS, TC_MEM, TC_MEM / 16>(s, R, ta, tb, th, tc, out);
}
__global__ void __launch_bounds__(TCW_M) tcw_grad_probe(const float* p, int R, const float* ta, const float* tb, const float* th, const float* tc, float* out) {
    extern __shared__ __align__(128) unsigned char probe_smem[];
    TcwSmem& s = *reinterpret_cast<TcwSmem*>(probe_smem);
    tcw_setup(s, p);
    grad_rounds<TcwSmem, TCW_M, TCW_M, TCW_M / 16>(s, R, ta, tb, th, tc, out);
}

// ---- one adjoint stage: forward<true> at y, backward<true> with cotangent L and weight wt, then the CTA's partial.
// Member m reads y[m][2], L[m][2], valid[m] and writes F[m][2], J[m][2].
__global__ void __launch_bounds__(TC_M) tc_stage_probe(const float* p, const float* y, const float* L, const int* valid, float wt,
                                                       float* F, float* J, float* partial) {
    extern __shared__ __align__(128) unsigned char probe_smem[];
    TcSmem& s = *reinterpret_cast<TcSmem*>(probe_smem);
    tc_setup(s, p);
    const int t = threadIdx.x, m = t & 31;
    TcState st;
    TcGrad g;
    g.zero();
    float H2q[16], f[2], j[2];
    tc_forward<true>(s, st, y[2 * m], y[2 * m + 1], f, H2q);
    tc_backward<true>(s, st, g, wt, L[2 * m], L[2 * m + 1], valid[m] != 0, H2q, j);
    if (t < TC_MEM) { F[2 * m] = f[0]; F[2 * m + 1] = f[1]; J[2 * m] = j[0]; J[2 * m + 1] = j[1]; }
    tc_grad_store(g, partial);
}
__global__ void __launch_bounds__(TCW_M) tcw_stage_probe(const float* p, const float* y, const float* L, const int* valid, float wt,
                                                         float* F, float* J, float* partial) {
    extern __shared__ __align__(128) unsigned char probe_smem[];
    TcwSmem& s = *reinterpret_cast<TcwSmem*>(probe_smem);
    tcw_setup(s, p);
    const int t = threadIdx.x;
    TcwState st;
    TcGrad g;
    g.zero();
    float H2[64], f[2], j[2];
    tcw_forward<true>(s, st, y[2 * t], y[2 * t + 1], f, H2);
    tcw_backward<true>(s, st, g, wt, L[2 * t], L[2 * t + 1], valid[t] != 0, H2, j);
    F[2 * t] = f[0]; F[2 * t + 1] = f[1]; J[2 * t] = j[0]; J[2 * t + 1] = j[1];
    tc_grad_store(g, partial);
}

template <class S, class K, class... A>
int launch(K kernel, A... args) {
    const int smem = (int)sizeof(S) + 128;
    cudaError_t e = cudaFuncSetAttribute(kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, smem);
    if (e != cudaSuccess) return (int)e;
    kernel<<<1, 128, smem>>>(args...);
    e = cudaGetLastError();
    if (e != cudaSuccess) return (int)e;
    return (int)cudaDeviceSynchronize();
}

}  // namespace

// wide = 0: the 32-member layout (TcSmem, D has 32 rows, a has 64); wide = 1: the 128-member layout (TcwSmem, 128 and 128)
extern "C" int probe_member_gemm(int wide, int tile_f, const float* p, const float* a, int w2t, float* D) {
    if (tile_f == TC_TB_F) return wide ? launch<TcwSmem>(tcw_member_probe<TC_TB_F>, p, a, w2t, D) : launch<TcSmem>(tc_member_probe<TC_TB_F>, p, a, w2t, D);
    if (tile_f == TC_TA_F) return wide ? launch<TcwSmem>(tcw_member_probe<TC_TA_F>, p, a, w2t, D) : launch<TcSmem>(tc_member_probe<TC_TA_F>, p, a, w2t, D);
    return (int)cudaErrorInvalidValue;
}
extern "C" int probe_grad_gemm(int wide, const float* p, int R, const float* ta, const float* tb, const float* th, const float* tc, float* out) {
    return wide ? launch<TcwSmem>(tcw_grad_probe, p, R, ta, tb, th, tc, out) : launch<TcSmem>(tc_grad_probe, p, R, ta, tb, th, tc, out);
}
extern "C" int probe_stage(int wide, const float* p, const float* y, const float* L, const int* valid, float wt, float* F, float* J, float* partial) {
    return wide ? launch<TcwSmem>(tcw_stage_probe, p, y, L, valid, wt, F, J, partial)
                : launch<TcSmem>(tc_stage_probe, p, y, L, valid, wt, F, J, partial);
}
