// mlp_tc_wide.cuh -- the WIDE layout of the tensor-core neural-ODE kernels (mlp_tc.cuh): one CTA = 128 ensemble members = the
// 128 rows (two M = 64 halves) of every MMA, one thread per member (64 tanh per layer and thread).  Highest throughput once
// every SM has work (N >= 2 x n_SM x 32 members); below that the 32-member layout of mlp_tc.cuh has 4x more CTAs and shorter
// stages.  The GEMMs, tiles and descriptors are those of mlp_tc.cuh (all 128 rows are distinct members here).
#pragma once
#include "mlp_tc.cuh"

namespace b200adj {

constexpr int TCW_M = 128;                                   // members per CTA

struct TcwSmem {
    alignas(128) unsigned char TA[TCW_M * TC_TA_F * 2];      // [member][wt dZ2 (64) | wt dZ1 (64)]
    alignas(128) unsigned char TH[TCW_M * TC_TA_F * 2];      // [member][H2 (64) | 1 | 0 ...]
    alignas(128) unsigned char TB[TCW_M * TC_TB_F * 2];      // [member][H1 (64) | y0 y1 1 | 0 ...]
    alignas(128) unsigned char TC[TCW_M * TC_TC_F * 2];      // [member][wt L0, wt L1 | 0 ...]
    alignas(128) unsigned char W2[64 * 64 * 2];             // (n = out i, k = in j)  = W2[i][j]
    alignas(128) unsigned char W2T[64 * 64 * 2];            // (n = in j,  k = out i) = W2[i][j]
    alignas(16) float D[TCW_M * TC_DP];                      // member-GEMM accumulator, fp32
    float W1a[64], W1b[64], b1[64], b2[64], W3a[64], W3b[64], b3[2];
};

struct TcwState {               // per-thread pipeline bookkeeping (identical in all threads)
    bool gpend = false;
};

__device__ __forceinline__ void tcw_setup(TcwSmem& s, const float* p) {
    const int t = threadIdx.x;
    for (int x = t; x < 64 * 64; x += TCW_M) {
        const int j = x / 64, i = x % 64;                                     // p[OW2 + j*64 + i] = W2[i][j]
        const __nv_bfloat16 w = __float2bfloat16(p[MLP_OW2 + x]);
        *reinterpret_cast<__nv_bfloat16*>(s.W2 + (i >> 3) * 1024 + (j >> 3) * 128 + (i & 7) * 16 + (j & 7) * 2) = w;
        *reinterpret_cast<__nv_bfloat16*>(s.W2T + (j >> 3) * 1024 + (i >> 3) * 128 + (j & 7) * 16 + (i & 7) * 2) = w;
    }
    if (t < 64) {
        s.W1a[t] = p[MLP_OW1 + t]; s.W1b[t] = p[MLP_OW1 + 64 + t]; s.b1[t] = p[MLP_OB1 + t]; s.b2[t] = p[MLP_OB2 + t];
        s.W3a[t] = p[MLP_OW3 + t * 2]; s.W3b[t] = p[MLP_OW3 + t * 2 + 1];
    }
    if (t < 2) s.b3[t] = p[MLP_OB3 + t];
    // constant parts of the tiles: TH features 64.. = [1, 0, ...], TB features 72..79 = 0, TC features 8..15 = 0
    const uint4 zero = make_uint4(0, 0, 0, 0);
    *tc_chunk<TC_TA_F>(s.TH, t, 8) = make_uint4(0x00003F80u, 0, 0, 0);       // bf16(1.0) = 0x3F80
#pragma unroll
    for (int kc = 9; kc < 16; kc++) *tc_chunk<TC_TA_F>(s.TH, t, kc) = zero;
    *tc_chunk<TC_TB_F>(s.TB, t, 8) = zero;
    *tc_chunk<TC_TB_F>(s.TB, t, 9) = zero;
    *tc_chunk<TC_TC_F>(s.TC, t, 0) = zero;
    *tc_chunk<TC_TC_F>(s.TC, t, 1) = zero;
    asm volatile("fence.proxy.async.shared::cta;" ::: "memory");
    __syncthreads();
}

__device__ __forceinline__ void tcw_wait_grad(TcwState& st) {
    if (st.gpend) { wgmma_wait_all(); st.gpend = false; }
}

// the member GEMM of this stage (A = the K-major tile a of 128 rows) staged to s.D as fp32, one M = 64 half at a time
__device__ __forceinline__ void tcw_member_mma(TcwSmem& s, const unsigned char* a, uint32_t a_sbo, const unsigned char* b) {
#pragma unroll 1
    for (int h = 0; h < 2; h++) {
        float d[32];
        tc_member_mma(d, smem_u32(a) + h * 8 * a_sbo, a_sbo, smem_u32(b));
        tc_stage(s.D, d, 64 * h);
    }
}

// F = f(y); leaves H1 (bf16) in this member's TB row and H2 in registers
template <bool GRAD>
__device__ __forceinline__ void tcw_forward(TcwSmem& s, TcwState& st, float y0, float y1, float* F, float* H2) {
    const int t = threadIdx.x;
    uint4 row[8];                                        // H1 of this member, bf16, computed while the previous stage's
#pragma unroll                                           // gradient GEMMs may still be reading the tiles
    for (int kc = 0; kc < 8; kc++) {
        float h[8];
#pragma unroll
        for (int q = 0; q < 8; q++) { const int j = kc * 8 + q; h[q] = tanh_fast(fmaf(s.W1a[j], y0, fmaf(s.W1b[j], y1, s.b1[j]))); }
        row[kc] = make_uint4(pack_bf16(h[0], h[1]), pack_bf16(h[2], h[3]), pack_bf16(h[4], h[5]), pack_bf16(h[6], h[7]));
    }
    if (GRAD) tcw_wait_grad(st);
#pragma unroll
    for (int kc = 0; kc < 8; kc++) *tc_chunk<TC_TB_F>(s.TB, t, kc) = row[kc];
    if (GRAD) *tc_chunk<TC_TB_F>(s.TB, t, 8) = make_uint4(pack_bf16(y0, y1), pack_bf16(1.0f, 0.0f), 0, 0);
    asm volatile("fence.proxy.async.shared::cta;" ::: "memory");
    __syncthreads();
    tcw_member_mma(s, s.TB, (TC_TB_F / 8) * 128, s.W2);
    __syncthreads();
    float f0 = s.b3[0], f1 = s.b3[1];
#pragma unroll
    for (int q4 = 0; q4 < 16; q4++) {
        const float4 z = *reinterpret_cast<const float4*>(s.D + t * TC_DP + 4 * q4);
        const float zz[4] = {z.x, z.y, z.z, z.w};
#pragma unroll
        for (int e = 0; e < 4; e++) {
            const int n = 4 * q4 + e;
            const float h2 = tanh_fast(zz[e] + s.b2[n]);
            H2[n] = h2;
            f0 = fmaf(s.W3a[n], h2, f0); f1 = fmaf(s.W3b[n], h2, f1);
        }
    }
    F[0] = f0; F[1] = f1;
}

// J = (df/dy)' L at the point of the last tcw_forward; issues the gradient GEMMs with weight wt (members with valid = false
// contribute nothing)
template <bool GRAD = true>
__device__ __forceinline__ void tcw_backward(TcwSmem& s, TcwState& st, TcGrad& g, float wt, float L0, float L1, bool valid, const float* H2, float* J) {
    const int t = threadIdx.x;
    const float wv = valid ? wt : 0.0f;
#pragma unroll
    for (int kc = 0; kc < 8; kc++) {
        float dz[8], hh[8];
#pragma unroll
        for (int q = 0; q < 8; q++) {
            const int n = kc * 8 + q;
            hh[q] = H2[n];
            dz[q] = wv * fmaf(s.W3a[n], L0, s.W3b[n] * L1) * (1.0f - hh[q] * hh[q]);
        }
        *tc_chunk<TC_TA_F>(s.TA, t, kc) = make_uint4(pack_bf16(dz[0], dz[1]), pack_bf16(dz[2], dz[3]), pack_bf16(dz[4], dz[5]), pack_bf16(dz[6], dz[7]));
        *tc_chunk<TC_TA_F>(s.TH, t, kc) = make_uint4(pack_bf16(hh[0], hh[1]), pack_bf16(hh[2], hh[3]), pack_bf16(hh[4], hh[5]), pack_bf16(hh[6], hh[7]));
    }
    *tc_chunk<TC_TC_F>(s.TC, t, 0) = make_uint4(pack_bf16(wv * L0, wv * L1), 0, 0, 0);
    asm volatile("fence.proxy.async.shared::cta;" ::: "memory");
    __syncthreads();
    tcw_member_mma(s, s.TA, (TC_TA_F / 8) * 128, s.W2T);
    __syncthreads();
    float j0 = 0.0f, j1 = 0.0f;
#pragma unroll
    for (int cb = 0; cb < 64; cb += 16) {
        float dz1[16];
#pragma unroll
        for (int half = 0; half < 2; half++) {
            const uint4 hv = *tc_chunk<TC_TB_F>(s.TB, t, cb / 8 + half);      // this member's H1 (bf16), features cb + 8 half ..
            const uint32_t hw[4] = {hv.x, hv.y, hv.z, hv.w};
            const float4 z0 = *reinterpret_cast<const float4*>(s.D + t * TC_DP + cb + 8 * half);
            const float4 z1 = *reinterpret_cast<const float4*>(s.D + t * TC_DP + cb + 8 * half + 4);
            const float zz[8] = {z0.x, z0.y, z0.z, z0.w, z1.x, z1.y, z1.z, z1.w};
#pragma unroll
            for (int q = 0; q < 8; q++) {
                const int j = cb + half * 8 + q;
                const float h1 = __uint_as_float((q & 1) ? (hw[q >> 1] & 0xFFFF0000u) : (hw[q >> 1] << 16));
                const float d = zz[q] * (1.0f - h1 * h1);      // wt dZ1
                dz1[half * 8 + q] = d;
                j0 = fmaf(s.W1a[j], d, j0); j1 = fmaf(s.W1b[j], d, j1);
            }
        }
        *tc_chunk<TC_TA_F>(s.TA, t, 8 + cb / 8) = make_uint4(pack_bf16(dz1[0], dz1[1]), pack_bf16(dz1[2], dz1[3]), pack_bf16(dz1[4], dz1[5]), pack_bf16(dz1[6], dz1[7]));
        *tc_chunk<TC_TA_F>(s.TA, t, 9 + cb / 8) = make_uint4(pack_bf16(dz1[8], dz1[9]), pack_bf16(dz1[10], dz1[11]), pack_bf16(dz1[12], dz1[13]), pack_bf16(dz1[14], dz1[15]));
    }
    const float inv = 1.0f / wt;
    J[0] = j0 * inv; J[1] = j1 * inv;
    asm volatile("fence.proxy.async.shared::cta;" ::: "memory");
    __syncthreads();
    if (GRAD) { tc_grad_mma<TCW_M / 16>(g, smem_u32(s.TA), smem_u32(s.TB), smem_u32(s.TH), smem_u32(s.TC)); st.gpend = true; }
}

// ---- forward ensemble solve (fixed-step Tsit5) ----
template <int UNUSED = 0>
__global__ void __launch_bounds__(TCW_M) mlp_tcw_forward_kernel(const __grid_constant__ MlpArgs<float> a) {
    extern __shared__ __align__(128) unsigned char tcw_smem_raw[];
    TcwSmem& s = *reinterpret_cast<TcwSmem*>(tcw_smem_raw);
    const int64_t N = a.N, base = (int64_t)blockIdx.x * TCW_M;
    const int t = threadIdx.x;
    const bool live = base + t < N;
    const int64_t col = live ? base + t : N - 1;
    tcw_setup(s, a.p);
    TcwState st;
    float u[2], kf[7][2], H2[64], F[2];
    u[0] = a.u0[col]; u[1] = a.u0[N + col];
    if (live) {
        a.ckpt[col] = u[0]; a.ckpt[N + col] = u[1];
        if (a.saved) { const int ks = a.save_of_step[0]; if (ks >= 0) { a.saved[((int64_t)ks * 2) * N + col] = u[0]; a.saved[((int64_t)ks * 2 + 1) * N + col] = u[1]; } }
    }
    tcw_forward<false>(s, st, u[0], u[1], kf[0], H2);
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
            tcw_forward<false>(s, st, y[0], y[1], F, H2);
            if (sg < 6) { kf[sg][0] = F[0]; kf[sg][1] = F[1]; }
        }
        if (live && a.kst) {
            // the dense forward solution of this step (k1..k6, k7 = f(u_{n+1})): the reverse pass reads it back instead of
            // repeating the six stage evaluations (6 of its 18 tensor-core round trips per step), 56 B per member-step
            float* ks_ = a.kst + ((int64_t)n * 14) * N + col;
#pragma unroll
            for (int j = 0; j < 6; j++) { ks_[(int64_t)(2 * j) * N] = kf[j][0]; ks_[(int64_t)(2 * j + 1) * N] = kf[j][1]; }
            ks_[(int64_t)12 * N] = F[0]; ks_[(int64_t)13 * N] = F[1];
        }
        u[0] = y[0]; u[1] = y[1]; kf[0][0] = F[0]; kf[0][1] = F[1];         // FSAL: f(u_{n+1})
        if (live) {
            a.ckpt[((int64_t)(n + 1) * 2) * N + col] = u[0]; a.ckpt[((int64_t)(n + 1) * 2 + 1) * N + col] = u[1];
            if (a.saved) { const int ks = a.save_of_step[n + 1]; if (ks >= 0) { a.saved[((int64_t)ks * 2) * N + col] = u[0]; a.saved[((int64_t)ks * 2 + 1) * N + col] = u[1]; } }
        }
    }
    if (live && a.status) a.status[col] = (isfinite(u[0]) && isfinite(u[1])) ? 0 : 1;
}

// ---- fused reverse pass (same stage sequence as mlp_reverse_kernel): InterpolatingAdjoint, or GaussAdjoint (GAUSS: seven
// adjoint stages without gradient GEMMs, then the gradient GEMMs at the three Gauss-Legendre nodes of the step, weight (h/2) w_g,
// accumulated in the same registers) ----
template <int COST, bool GAUSS = false>
__global__ void __launch_bounds__(TCW_M) mlp_tcw_reverse_kernel(const __grid_constant__ MlpArgs<float> a) {
    extern __shared__ __align__(128) unsigned char tcw_smem_raw[];
    TcwSmem& s = *reinterpret_cast<TcwSmem*>(tcw_smem_raw);
    const int64_t N = a.N, base = (int64_t)blockIdx.x * TCW_M;
    const int t = threadIdx.x;
    const bool live = base + t < N;
    const int64_t col = live ? base + t : N - 1;
    const Tsit5Tables& tb = a.tb;
    tcw_setup(s, a.p);
    TcwState st;
    TcGrad g;
    g.zero();
    float lam[2] = {0.0f, 0.0f}, uhi[2], ulo[2], kf[7][2], ka[7][2], H2[64], F[2], J[2];
    auto cotangent = [&](int ks, const float* yy) {
        if (COST == COST_EXPLICIT) { lam[0] += a.dLdu[((int64_t)ks * 2) * N + col]; lam[1] += a.dLdu[((int64_t)ks * 2 + 1) * N + col]; }
        else { lam[0] += (float)(a.cost_a[0] * (double)yy[0] + a.cost_b[0]); lam[1] += (float)(a.cost_a[1] * (double)yy[1] + a.cost_b[1]); }
    };
    uhi[0] = a.ckpt[((int64_t)a.S * 2) * N + col]; uhi[1] = a.ckpt[((int64_t)a.S * 2 + 1) * N + col];
    { const int ks = a.save_of_step[a.S]; if (ks >= 0) cotangent(ks, uhi); }
    if (!a.kst) tcw_forward<true>(s, st, uhi[0], uhi[1], kf[6], H2);    // f(u_S) = forward k7 of the last step
    for (int n = a.S - 1; n >= 0; n--) {
        ulo[0] = a.ckpt[((int64_t)n * 2) * N + col]; ulo[1] = a.ckpt[((int64_t)n * 2 + 1) * N + col];
        // ---- forward stages k1..k7 of [t_n, t_{n+1}]: read back from the forward pass (a.kst) or recomputed ----
        if (a.kst) {
            const float* ks_ = a.kst + ((int64_t)n * 14) * N + col;
#pragma unroll
            for (int j = 0; j < 7; j++) { kf[j][0] = ks_[(int64_t)(2 * j) * N]; kf[j][1] = ks_[(int64_t)(2 * j + 1) * N]; }
        } else {
            tcw_forward<true>(s, st, ulo[0], ulo[1], kf[0], H2);
#pragma unroll 1
            for (int sg = 1; sg <= 5; sg++) {
                float y[2];
#pragma unroll
                for (int c = 0; c < 2; c++) {
                    double acc = (double)ulo[c];
                    for (int j = 0; j < sg; j++) acc = fma(tb.hA[sg][j], (double)kf[j][c], acc);
                    y[c] = (float)acc;
                }
                tcw_forward<true>(s, st, y[0], y[1], kf[sg], H2);
            }
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
            tcw_forward<true>(s, st, y[0], y[1], F, H2);
            if (GAUSS) tcw_backward<false>(s, st, g, 1.0f, L[0], L[1], live, H2, J);
            else tcw_backward<true>(s, st, g, (float)tb.hA[6][sg], L[0], L[1], live, H2, J);
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
                tcw_forward<true>(s, st, y[0], y[1], F, H2);
                tcw_backward<true>(s, st, g, (float)tb.hGW[gq], L[0], L[1], live, H2, J);
            }
        }
#pragma unroll
        for (int c = 0; c < 2; c++) {
            double l = (double)lam[c];
            for (int j = 0; j < 6; j++) l = fma(tb.hA[6][j], (double)ka[j][c], l);
            lam[c] = (float)l;
        }
        { const int ks = a.save_of_step[n]; if (ks >= 0 && !((a.flags & 1u) && n == 0)) cotangent(ks, ulo); }
        uhi[0] = ulo[0]; uhi[1] = ulo[1];
        if (!a.kst) { kf[6][0] = kf[0][0]; kf[6][1] = kf[0][1]; }
    }
    if (live) { a.du0[col] = lam[0]; a.du0[N + col] = lam[1]; }
    // ---- parameter gradient of this CTA out of the accumulator fragments ----
    tc_grad_store(g, a.partials + (int64_t)blockIdx.x * MLP_P);
}

}  // namespace b200adj
