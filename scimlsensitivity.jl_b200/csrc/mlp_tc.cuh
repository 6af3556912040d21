// mlp_tc.cuh -- the neural-ODE family (BASELINE config C4, dtype BF16_F32ACC) with EVERY GEMM-shaped piece of the time loop on
// the Hopper tensor cores: bf16 operands in shared memory, fp32 accumulators in the registers of the CTA's one warpgroup,
// wgmma.mma_async issued by all 128 threads, no operand tapes and no reduction over members on the CUDA cores.
//
// Narrow layout (at the BASELINE size N = 4096, one member per thread would be 32 CTAs on 132 SMs, each a serial chain of
// 128 x 128 MUFU.TANH + MMA round trips per stage):
//   one CTA = 32 ensemble members x 4 warps.  Thread (w, m) = warp w, lane m owns member m's feature QUARTER [16 w, 16 w + 16):
//   16 tanh per layer instead of 64, 128 CTAs at N = 4096, several CTAs per SM at large N.  The member MMAs have M = 64 rows:
//   rows 0..31 are the members, rows 32..63 stay zero.  The accumulator fragment of rows 0..31 (warps 0 and 1) goes through a
//   shared fp32 tile, from which thread (w, m) reads member m's columns 16 w ..  The member state (u, lam, RK stages, d = 2)
//   is kept redundantly by the 4 threads of a member; the two 2-vectors a stage returns (f, J'lam) are summed over the
//   quarters through shared memory.
//
//   member GEMMs (M = 64, N = 64, K = 64; K-major operands):
//     forward   Z2 = H1 W2'          A = tile TB (H1),      B = W2   (n = out, k = in)
//     backward  dH1 = dZ2 W2         A = tile TA (wt dZ2),  B = W2^T (n = in,  k = out)
//   gradient GEMMs (K = the 32 members; the SAME tiles read as MN-major operands -- element (m, f) of a member tile sits at
//   (m/8) ROW + (f/8) 128 + (m%8) 16 + (f%8) 2, which is at once the canonical K-major layout of [member x feature] and the
//   canonical MN-major layout of [feature x member]), accumulated in registers over the whole reverse pass (two M = 64 halves):
//     G1 [128 x 80] += [wt dZ2 | wt dZ1]' [H1 | y0 y1 1 | 0]   ->  dW2, db2 (rows 0..63), dW1, db1 (rows 64..127)
//     G2 [128 x 16] += [H2 | 1 | 0]' [wt L0, wt L1 | 0]        ->  dW3' (rows 0..63), db3 (row 64)
//   wt = h b_j is folded into the cotangent side before the bf16 rounding; the backward member GEMM is linear, so the
//   vector-Jacobian product is recovered by dividing by wt.  The gradient GEMMs of a stage run asynchronously until the next
//   stage's H1 is ready to be written.
//
// Per adjoint stage: 2 member GEMMs (4 MMAs each) + 2 gradient GEMMs (4 MMAs each); per forward stage: 1 member GEMM.
// tanh is the hardware tanh.approx.f32 (relative error 2^-11, below the bf16 rounding of the operands).
// Reference functions replaced: as mlp.cuh (sense functor, split_states, vecjacobian!, ReverseLossCallback).
#pragma once
#include <cuda_bf16.h>
#include <cuda_runtime.h>
#include <stdint.h>
#include "mlp.cuh"
#include "wgmma.cuh"

namespace b200adj {

constexpr int TC_MEM = 32;                                  // members per CTA
constexpr int TC_M = 128;                                   // threads per CTA (one warpgroup)
constexpr int TC_ROWS = 64;                                 // rows of the member MMAs: 32 members, 32 zero rows
constexpr int TC_TA_F = 128, TC_TB_F = 80, TC_TC_F = 16;      // feature widths of the tiles
constexpr int TC_DP = 68;                                   // pitch (floats) of the fp32 accumulator staging tile

struct TcSmem {
    alignas(128) unsigned char TA[TC_ROWS * TC_TA_F * 2];   // [row][wt dZ2 (64) | wt dZ1 (64)]
    alignas(128) unsigned char TH[TC_MEM * TC_TA_F * 2];    // [member][H2 (64) | 1 | 0 ...]
    alignas(128) unsigned char TB[TC_ROWS * TC_TB_F * 2];   // [row][H1 (64) | y0 y1 1 | 0 ...]
    alignas(128) unsigned char TC[TC_MEM * TC_TC_F * 2];    // [member][wt L0, wt L1 | 0 ...]
    alignas(128) unsigned char W2[64 * 64 * 2];             // (n = out i, k = in j)  = W2[i][j]
    alignas(128) unsigned char W2T[64 * 64 * 2];            // (n = in j,  k = out i) = W2[i][j]
    alignas(16) float D[TC_MEM * TC_DP];                     // member-GEMM accumulator rows 0..31, fp32
    float W1a[64], W1b[64], b1[64], b2[64], W3a[64], W3b[64], b3[2];
    float red[2][4][TC_MEM][2];                             // per-quarter partial sums of the 2-vectors a stage returns (double-buffered)
};

__device__ __forceinline__ float tanh_fast(float x) { float y; asm("tanh.approx.f32 %0, %1;" : "=f"(y) : "f"(x)); return y; }
__device__ __forceinline__ uint32_t pack_bf16(float a, float b) { __nv_bfloat162 v = __floats2bfloat162_rn(a, b); return *reinterpret_cast<uint32_t*>(&v); }
// 16-byte chunk kc (features 8 kc .. 8 kc + 7) of row r in a tile of F features
template <int F> __device__ __forceinline__ uint4* tc_chunk(unsigned char* tile, int r, int kc) {
    return reinterpret_cast<uint4*>(tile + (r >> 3) * (F / 8) * 128 + kc * 128 + (r & 7) * 16);
}

struct TcState {               // per-thread pipeline bookkeeping (identical in all threads)
    uint32_t rb = 0;
    bool gpend = false;
};

// the gradient accumulators G1 (two M = 64 halves x N = 80) and G2 (two halves x N = 16), wgmma fragments
struct TcGrad {
    float g1[2][40], g2[2][8];
    __device__ __forceinline__ void zero() {
#pragma unroll
        for (int h = 0; h < 2; h++) {
#pragma unroll
            for (int i = 0; i < 40; i++) g1[h][i] = 0.0f;
#pragma unroll
            for (int i = 0; i < 8; i++) g2[h][i] = 0.0f;
        }
    }
};

// d = A[64 x 64] B', A = rows 0..63 of a K-major tile (8-row groups a_sbo bytes apart), B = a K-major 64 x 64 weight tile
__device__ __forceinline__ void tc_member_mma(float (&d)[32], uint32_t a, uint32_t a_sbo, uint32_t b) {
    wgmma_fence();
#pragma unroll
    for (int k = 0; k < 4; k++) wgmma_m64n64<0, 0>(d, wgmma_desc(a + k * 256, 128, a_sbo), wgmma_desc(b + k * 256, 128, 1024), k > 0);
    wgmma_commit();
    wgmma_wait_all();
    wgmma_fence_operand(d);
}
// the fragment of d (rows row0 + 0..63) into the fp32 staging tile of pitch TC_DP
__device__ __forceinline__ void tc_stage(float* D, const float (&d)[32], int row0) {
    const int w = (threadIdx.x >> 5) & 3, l = threadIdx.x & 31, r = row0 + 16 * w + (l >> 2), c = 2 * (l & 3);
#pragma unroll
    for (int j = 0; j < 8; j++) {
        *reinterpret_cast<float2*>(D + r * TC_DP + 8 * j + c) = make_float2(d[4 * j], d[4 * j + 1]);
        *reinterpret_cast<float2*>(D + (r + 8) * TC_DP + 8 * j + c) = make_float2(d[4 * j + 2], d[4 * j + 3]);
    }
}
// G1 += TA' TB, G2 += TH' TC over the first 16 KS member rows of the tiles (asynchronous: tc_wait_grad before the tiles change)
template <int KS>
__device__ __forceinline__ void tc_grad_mma(TcGrad& g, uint32_t TA, uint32_t TB, uint32_t TH, uint32_t TC) {
    constexpr uint32_t SA = (TC_TA_F / 8) * 128, SB = (TC_TB_F / 8) * 128, SC = (TC_TC_F / 8) * 128;
    wgmma_fence();
#pragma unroll
    for (int h = 0; h < 2; h++)
#pragma unroll
        for (int k = 0; k < KS; k++)       // K = 16 members per MMA = 2 member groups of 8
            wgmma_m64n80<1, 1>(g.g1[h], wgmma_desc(TA + h * 1024 + k * 2 * SA, SA, 128), wgmma_desc(TB + k * 2 * SB, SB, 128), 1u);
#pragma unroll
    for (int h = 0; h < 2; h++)
#pragma unroll
        for (int k = 0; k < KS; k++)
            wgmma_m64n16<1, 1>(g.g2[h], wgmma_desc(TH + h * 1024 + k * 2 * SA, SA, 128), wgmma_desc(TC + k * 2 * SC, SC, 128), 1u);
    wgmma_commit();
}
// this CTA's parameter gradient out of the G1 / G2 fragments
__device__ __forceinline__ void tc_grad_store(TcGrad& g, float* out) {
    wgmma_wait_all();
#pragma unroll
    for (int h = 0; h < 2; h++) { wgmma_fence_operand(g.g1[h]); wgmma_fence_operand(g.g2[h]); }
    const int w = (threadIdx.x >> 5) & 3, l = threadIdx.x & 31;
#pragma unroll
    for (int i = 0; i < 40; i++) {
        const int r = 16 * w + (l >> 2) + 8 * ((i >> 1) & 1), c = 8 * (i >> 2) + 2 * (l & 3) + (i & 1);
        if (c < 64) out[MLP_OW2 + c * 64 + r] = g.g1[0][i];      // row i = r: dW2[i][c], db2[i] (c = 66)
        else if (c == 66) out[MLP_OB2 + r] = g.g1[0][i];
        if (c == 64) out[MLP_OW1 + r] = g.g1[1][i];               // row 64 + j: dW1[j][c - 64], db1[j] (c = 66)
        else if (c == 65) out[MLP_OW1 + 64 + r] = g.g1[1][i];
        else if (c == 66) out[MLP_OB1 + r] = g.g1[1][i];
    }
#pragma unroll
    for (int i = 0; i < 8; i++) {
        const int r = 16 * w + (l >> 2) + 8 * ((i >> 1) & 1), c = 8 * (i >> 2) + 2 * (l & 3) + (i & 1);
        if (c < 2) {
            out[MLP_OW3 + r * 2 + c] = g.g2[0][i];                 // dW3[c][n = r]
            if (r == 0) out[MLP_OB3 + c] = g.g2[1][i];             // row 64: db3
        }
    }
}

__device__ __forceinline__ void tc_setup(TcSmem& s, const float* p) {
    const int t = threadIdx.x, m = t & 31, w = t >> 5;
    for (int x = t; x < 64 * 64; x += TC_M) {
        const int j = x / 64, i = x % 64;                                     // p[OW2 + j*64 + i] = W2[i][j]
        const __nv_bfloat16 wv = __float2bfloat16(p[MLP_OW2 + x]);
        *reinterpret_cast<__nv_bfloat16*>(s.W2 + (i >> 3) * 1024 + (j >> 3) * 128 + (i & 7) * 16 + (j & 7) * 2) = wv;
        *reinterpret_cast<__nv_bfloat16*>(s.W2T + (j >> 3) * 1024 + (i >> 3) * 128 + (j & 7) * 16 + (i & 7) * 2) = wv;
    }
    if (t < 64) {
        s.W1a[t] = p[MLP_OW1 + t]; s.W1b[t] = p[MLP_OW1 + 64 + t]; s.b1[t] = p[MLP_OB1 + t]; s.b2[t] = p[MLP_OB2 + t];
        s.W3a[t] = p[MLP_OW3 + t * 2]; s.W3b[t] = p[MLP_OW3 + t * 2 + 1];
    }
    if (t < 2) s.b3[t] = p[MLP_OB3 + t];
    // constant parts of the tiles: TH features 64.. = [1, 0, ...], TB features 64..79 = 0 (y, 1 written per stage), TC = 0,
    // TA / TB rows 32..63 = 0 (the unused rows of the member MMAs)
    const uint4 zero = make_uint4(0, 0, 0, 0);
    *tc_chunk<TC_TA_F>(s.TH, m, 8 + 2 * w) = w == 0 ? make_uint4(0x00003F80u, 0, 0, 0) : zero;       // bf16(1.0) = 0x3F80
    *tc_chunk<TC_TA_F>(s.TH, m, 9 + 2 * w) = zero;
    if (w == 0) { *tc_chunk<TC_TB_F>(s.TB, m, 8) = zero; *tc_chunk<TC_TB_F>(s.TB, m, 9) = zero; }
    if (w == 0) { *tc_chunk<TC_TC_F>(s.TC, m, 0) = zero; *tc_chunk<TC_TC_F>(s.TC, m, 1) = zero; }
    if (w == 2) {
        const int r = 32 + m;                                                  // rows 32..63
#pragma unroll
        for (int kc = 0; kc < TC_TB_F / 8; kc++) *tc_chunk<TC_TB_F>(s.TB, r, kc) = zero;
#pragma unroll
        for (int kc = 0; kc < TC_TA_F / 8; kc++) *tc_chunk<TC_TA_F>(s.TA, r, kc) = zero;
    }
    asm volatile("fence.proxy.async.shared::cta;" ::: "memory");
    __syncthreads();
}

// the previous stage's gradient GEMMs read ALL rows of the tiles, and wgmma.wait_group only covers the executing thread's
// part of them: every warp's wait must have returned (the barrier) before any thread overwrites a tile row
__device__ __forceinline__ void tc_wait_grad(TcState& st) {
    if (st.gpend) { wgmma_wait_all(); __syncthreads(); st.gpend = false; }
}

// F = f(y) for this thread's member; leaves H1 (bf16) in TB and this thread's H2 quarter in registers
template <bool GRAD>
__device__ __forceinline__ void tc_forward(TcSmem& s, TcState& st, float y0, float y1, float* F, float* H2q) {
    const int t = threadIdx.x, m = t & 31, w = t >> 5;
    uint4 row[2];                                        // this thread's H1 quarter, bf16, computed while the previous stage's
#pragma unroll                                           // gradient GEMMs may still be reading the tiles
    for (int c = 0; c < 2; c++) {
        float h[8];
#pragma unroll
        for (int q = 0; q < 8; q++) { const int j = 16 * w + 8 * c + q; h[q] = tanh_fast(fmaf(s.W1a[j], y0, fmaf(s.W1b[j], y1, s.b1[j]))); }
        row[c] = make_uint4(pack_bf16(h[0], h[1]), pack_bf16(h[2], h[3]), pack_bf16(h[4], h[5]), pack_bf16(h[6], h[7]));
    }
    if (GRAD) tc_wait_grad(st);
    *tc_chunk<TC_TB_F>(s.TB, m, 2 * w) = row[0];
    *tc_chunk<TC_TB_F>(s.TB, m, 2 * w + 1) = row[1];
    if (GRAD && w == 0) *tc_chunk<TC_TB_F>(s.TB, m, 8) = make_uint4(pack_bf16(y0, y1), pack_bf16(1.0f, 0.0f), 0, 0);
    asm volatile("fence.proxy.async.shared::cta;" ::: "memory");
    __syncthreads();
    {
        float d[32];
        tc_member_mma(d, smem_u32(s.TB), (TC_TB_F / 8) * 128, smem_u32(s.W2));
        if (w < 2) tc_stage(s.D, d, 0);
    }
    __syncthreads();
    float f0 = 0.0f, f1 = 0.0f;
#pragma unroll
    for (int q4 = 0; q4 < 4; q4++) {
        const float4 z = *reinterpret_cast<const float4*>(s.D + m * TC_DP + 16 * w + 4 * q4);     // member m, columns 16 w ..
        const float zz[4] = {z.x, z.y, z.z, z.w};
#pragma unroll
        for (int e = 0; e < 4; e++) {
            const int q = 4 * q4 + e, n = 16 * w + q;
            const float h2 = tanh_fast(zz[e] + s.b2[n]);
            H2q[q] = h2;
            f0 = fmaf(s.W3a[n], h2, f0); f1 = fmaf(s.W3b[n], h2, f1);
        }
    }
    // sum over the four feature quarters (fixed order => all four threads of a member hold the same bits)
    float (*red)[TC_MEM][2] = s.red[st.rb]; st.rb ^= 1;
    red[w][m][0] = f0; red[w][m][1] = f1;
    __syncthreads();
    F[0] = s.b3[0] + ((red[0][m][0] + red[1][m][0]) + (red[2][m][0] + red[3][m][0]));
    F[1] = s.b3[1] + ((red[0][m][1] + red[1][m][1]) + (red[2][m][1] + red[3][m][1]));
}

// J = (df/dy)' L at the point of the last tc_forward; issues the gradient GEMMs with weight wt (members with valid = false
// contribute nothing)
template <bool GRAD = true>
__device__ __forceinline__ void tc_backward(TcSmem& s, TcState& st, TcGrad& g, float wt, float L0, float L1, bool valid, const float* H2q, float* J) {
    const int t = threadIdx.x, m = t & 31, w = t >> 5;
    const float wv = valid ? wt : 0.0f;
    uint4 dzc[2], hhc[2];
#pragma unroll
    for (int c = 0; c < 2; c++) {
        float dz[8], hh[8];
#pragma unroll
        for (int q = 0; q < 8; q++) {
            const int n = 16 * w + 8 * c + q;
            hh[q] = H2q[8 * c + q];
            dz[q] = wv * fmaf(s.W3a[n], L0, s.W3b[n] * L1) * (1.0f - hh[q] * hh[q]);
        }
        dzc[c] = make_uint4(pack_bf16(dz[0], dz[1]), pack_bf16(dz[2], dz[3]), pack_bf16(dz[4], dz[5]), pack_bf16(dz[6], dz[7]));
        hhc[c] = make_uint4(pack_bf16(hh[0], hh[1]), pack_bf16(hh[2], hh[3]), pack_bf16(hh[4], hh[5]), pack_bf16(hh[6], hh[7]));
    }
    *tc_chunk<TC_TA_F>(s.TA, m, 2 * w) = dzc[0];
    *tc_chunk<TC_TA_F>(s.TA, m, 2 * w + 1) = dzc[1];
    *tc_chunk<TC_TA_F>(s.TH, m, 2 * w) = hhc[0];
    *tc_chunk<TC_TA_F>(s.TH, m, 2 * w + 1) = hhc[1];
    if (w == 0) *tc_chunk<TC_TC_F>(s.TC, m, 0) = make_uint4(pack_bf16(wv * L0, wv * L1), 0, 0, 0);
    asm volatile("fence.proxy.async.shared::cta;" ::: "memory");
    __syncthreads();
    {
        float d[32];
        tc_member_mma(d, smem_u32(s.TA), (TC_TA_F / 8) * 128, smem_u32(s.W2T));
        if (w < 2) tc_stage(s.D, d, 0);
    }
    __syncthreads();
    float j0 = 0.0f, j1 = 0.0f;
    {
        float dz1[16];
#pragma unroll
        for (int c = 0; c < 2; c++) {
            const uint4 hv = *tc_chunk<TC_TB_F>(s.TB, m, 2 * w + c);      // this member's H1 (bf16), features 16 w + 8 c ..
            const uint32_t hw[4] = {hv.x, hv.y, hv.z, hv.w};
            const float4 z0 = *reinterpret_cast<const float4*>(s.D + m * TC_DP + 16 * w + 8 * c);
            const float4 z1 = *reinterpret_cast<const float4*>(s.D + m * TC_DP + 16 * w + 8 * c + 4);
            const float zz[8] = {z0.x, z0.y, z0.z, z0.w, z1.x, z1.y, z1.z, z1.w};
#pragma unroll
            for (int q = 0; q < 8; q++) {
                const int j = 16 * w + 8 * c + q;
                const float h1 = __uint_as_float((q & 1) ? (hw[q >> 1] & 0xFFFF0000u) : (hw[q >> 1] << 16));
                const float d = zz[q] * (1.0f - h1 * h1);      // wt dZ1
                dz1[8 * c + q] = d;
                j0 = fmaf(s.W1a[j], d, j0); j1 = fmaf(s.W1b[j], d, j1);
            }
        }
        *tc_chunk<TC_TA_F>(s.TA, m, 8 + 2 * w) = make_uint4(pack_bf16(dz1[0], dz1[1]), pack_bf16(dz1[2], dz1[3]), pack_bf16(dz1[4], dz1[5]), pack_bf16(dz1[6], dz1[7]));
        *tc_chunk<TC_TA_F>(s.TA, m, 9 + 2 * w) = make_uint4(pack_bf16(dz1[8], dz1[9]), pack_bf16(dz1[10], dz1[11]), pack_bf16(dz1[12], dz1[13]), pack_bf16(dz1[14], dz1[15]));
    }
    float (*red)[TC_MEM][2] = s.red[st.rb]; st.rb ^= 1;
    red[w][m][0] = j0; red[w][m][1] = j1;
    asm volatile("fence.proxy.async.shared::cta;" ::: "memory");
    __syncthreads();
    const float inv = 1.0f / wt;
    J[0] = ((red[0][m][0] + red[1][m][0]) + (red[2][m][0] + red[3][m][0])) * inv;
    J[1] = ((red[0][m][1] + red[1][m][1]) + (red[2][m][1] + red[3][m][1])) * inv;
    if (GRAD) { tc_grad_mma<TC_MEM / 16>(g, smem_u32(s.TA), smem_u32(s.TB), smem_u32(s.TH), smem_u32(s.TC)); st.gpend = true; }
}

// ---- forward ensemble solve (fixed-step Tsit5) ----
template <int UNUSED = 0>
__global__ void __launch_bounds__(TC_M) mlp_tc_forward_kernel(const __grid_constant__ MlpArgs<float> a) {
    extern __shared__ __align__(128) unsigned char tc_smem_raw[];
    TcSmem& s = *reinterpret_cast<TcSmem*>(tc_smem_raw);
    const int64_t N = a.N, base = (int64_t)blockIdx.x * TC_MEM;
    const int t = threadIdx.x, m = t & 31;
    const bool live = base + m < N, writer = live && (t >> 5) == 0;        // one of the four threads of a member stores
    const int64_t col = live ? base + m : N - 1;
    tc_setup(s, a.p);
    TcState st;
    float u[2], kf[7][2], H2q[16], F[2];
    u[0] = a.u0[col]; u[1] = a.u0[N + col];
    if (writer) {
        a.ckpt[col] = u[0]; a.ckpt[N + col] = u[1];
        if (a.saved) { const int ks = a.save_of_step[0]; if (ks >= 0) { a.saved[((int64_t)ks * 2) * N + col] = u[0]; a.saved[((int64_t)ks * 2 + 1) * N + col] = u[1]; } }
    }
    tc_forward<false>(s, st, u[0], u[1], kf[0], H2q);
    for (int n = 0; n < a.S; n++) {
        float y[2];
#pragma unroll 1
        for (int sg = 1; sg <= 6; sg++) {
#pragma unroll
            for (int c = 0; c < 2; c++) {
                double acc = (double)u[c];
                for (int j = 0; j < sg; j++) acc = fma(a.tb.hA[sg][j], (double)kf[j][c], acc);
                y[c] = (float)acc;
            }
            tc_forward<false>(s, st, y[0], y[1], F, H2q);
            if (sg < 6) { kf[sg][0] = F[0]; kf[sg][1] = F[1]; }
        }
        if (writer) {
            // the dense forward solution of this step (k1..k6, k7 = f(u_{n+1})): the reverse pass reads it back instead of
            // repeating the six stage evaluations (6 of its 18 tensor-core round trips per step), 56 B per member-step
            float* ks_ = a.kst + ((int64_t)n * 14) * N + col;
#pragma unroll
            for (int j = 0; j < 6; j++) { ks_[(int64_t)(2 * j) * N] = kf[j][0]; ks_[(int64_t)(2 * j + 1) * N] = kf[j][1]; }
            ks_[(int64_t)12 * N] = F[0]; ks_[(int64_t)13 * N] = F[1];
        }
        u[0] = y[0]; u[1] = y[1]; kf[0][0] = F[0]; kf[0][1] = F[1];         // FSAL: f(u_{n+1})
        if (writer) {
            a.ckpt[((int64_t)(n + 1) * 2) * N + col] = u[0]; a.ckpt[((int64_t)(n + 1) * 2 + 1) * N + col] = u[1];
            if (a.saved) { const int ks = a.save_of_step[n + 1]; if (ks >= 0) { a.saved[((int64_t)ks * 2) * N + col] = u[0]; a.saved[((int64_t)ks * 2 + 1) * N + col] = u[1]; } }
        }
    }
    if (writer && a.status) a.status[col] = (isfinite(u[0]) && isfinite(u[1])) ? 0 : 1;
}

// ---- fused reverse pass (same stage sequence as mlp_reverse_kernel): InterpolatingAdjoint, or GaussAdjoint (GAUSS: seven
// adjoint stages without gradient GEMMs, then the gradient GEMMs at the three Gauss-Legendre nodes of the step, weight (h/2) w_g,
// accumulated in the same registers) ----
template <int COST, bool GAUSS = false>
__global__ void __launch_bounds__(TC_M) mlp_tc_reverse_kernel(const __grid_constant__ MlpArgs<float> a) {
    extern __shared__ __align__(128) unsigned char tc_smem_raw[];
    TcSmem& s = *reinterpret_cast<TcSmem*>(tc_smem_raw);
    const int64_t N = a.N, base = (int64_t)blockIdx.x * TC_MEM;
    const int t = threadIdx.x, m = t & 31;
    const bool live = base + m < N, writer = live && (t >> 5) == 0;
    const int64_t col = live ? base + m : N - 1;
    const Tsit5Tables& tb = a.tb;
    tc_setup(s, a.p);
    TcState st;
    TcGrad g;
    g.zero();
    float lam[2] = {0.0f, 0.0f}, uhi[2], ulo[2], kf[7][2], ka[7][2], H2q[16], F[2], J[2];
    auto cotangent = [&](int ks, const float* yy) {
        if (COST == COST_EXPLICIT) { lam[0] += a.dLdu[((int64_t)ks * 2) * N + col]; lam[1] += a.dLdu[((int64_t)ks * 2 + 1) * N + col]; }
        else { lam[0] += (float)(a.cost_a[0] * (double)yy[0] + a.cost_b[0]); lam[1] += (float)(a.cost_a[1] * (double)yy[1] + a.cost_b[1]); }
    };
    uhi[0] = a.ckpt[((int64_t)a.S * 2) * N + col]; uhi[1] = a.ckpt[((int64_t)a.S * 2 + 1) * N + col];
    { const int ks = a.save_of_step[a.S]; if (ks >= 0) cotangent(ks, uhi); }
    for (int n = a.S - 1; n >= 0; n--) {
        ulo[0] = a.ckpt[((int64_t)n * 2) * N + col]; ulo[1] = a.ckpt[((int64_t)n * 2 + 1) * N + col];
        // ---- forward stages k1..k7 of [t_n, t_{n+1}]: read back from the forward pass ----
        {
            const float* ks_ = a.kst + ((int64_t)n * 14) * N + col;
#pragma unroll
            for (int j = 0; j < 7; j++) { kf[j][0] = ks_[(int64_t)(2 * j) * N]; kf[j][1] = ks_[(int64_t)(2 * j + 1) * N]; }
        }
        // ---- adjoint stages 0..5 (GaussAdjoint: 0..6, the 7th derivative feeds the dense output of the adjoint step) ----
#pragma unroll 1
        for (int sg = 0; sg <= (GAUSS ? 6 : 5); sg++) {
            float L[2], y[2];
#pragma unroll
            for (int c = 0; c < 2; c++) {
                double l = (double)lam[c];
                for (int j = 0; j < sg && j < 6; j++) l = fma(tb.hA[sg][j], (double)ka[j][c], l);
                L[c] = (float)l;
                double yv;
                if (sg == 0) yv = (double)uhi[c];
                else if (sg >= 5) yv = (double)ulo[c];
                else { yv = (double)ulo[c]; for (int j = 0; j < 7; j++) yv = fma(tb.hBst[sg - 1][j], (double)kf[j][c], yv); }
                y[c] = (float)yv;
            }
            tc_forward<true>(s, st, y[0], y[1], F, H2q);
            if (GAUSS) tc_backward<false>(s, st, g, 1.0f, L[0], L[1], live, H2q, J);
            else tc_backward<true>(s, st, g, (float)tb.hA[6][sg], L[0], L[1], live, H2q, J);
            ka[sg][0] = J[0]; ka[sg][1] = J[1];
        }
        if (GAUSS) {
#pragma unroll 1
            for (int gq = 0; gq < 3; gq++) {
                float L[2], y[2];
#pragma unroll
                for (int c = 0; c < 2; c++) {
                    double l = (double)lam[c], yv = (double)ulo[c];
                    for (int j = 0; j < 7; j++) { l = fma(tb.hBq[gq][j], (double)ka[j][c], l); yv = fma(tb.hBq[2 - gq][j], (double)kf[j][c], yv); }
                    L[c] = (float)l; y[c] = (float)yv;
                }
                tc_forward<true>(s, st, y[0], y[1], F, H2q);
                tc_backward<true>(s, st, g, (float)tb.hGW[gq], L[0], L[1], live, H2q, J);
            }
        }
#pragma unroll
        for (int c = 0; c < 2; c++) {
            double l = (double)lam[c];
            for (int j = 0; j < 6; j++) l = fma(tb.hA[6][j], (double)ka[j][c], l);
            lam[c] = (float)l;
        }
        { const int ks = a.save_of_step[n]; if (ks >= 0 && !((a.flags & KF_NO_START) && n == 0)) cotangent(ks, ulo); }
        uhi[0] = ulo[0]; uhi[1] = ulo[1];
    }
    if (writer) { a.du0[col] = lam[0]; a.du0[N + col] = lam[1]; }
    // ---- parameter gradient of this CTA out of the accumulator fragments ----
    tc_grad_store(g, a.partials + (int64_t)blockIdx.x * MLP_P);
}

}  // namespace b200adj
