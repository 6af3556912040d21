// mlp.cuh -- Neural-ODE family  f(u) = W3 tanh(W2 tanh(W1 u + b1) + b2) + b3,  2 -> 64 -> 64 -> 2 (BASELINE config C4),
// shared parameters, InterpolatingAdjoint with fixed-step Tsit5.
//
// Batched-state formulation (SURVEY.md 7.2 item 6 / "within-ODE batching", docs/src/tutorials/data_parallel.md:11-75):
// a thread block owns a tile of TB ensemble members, activations live in shared memory as [64][TB] matrices, every dense
// layer is a [64 x 64] x [64 x TB] register-tiled product, and the parameter gradient  mu += h b_j F(y_j)' lam_j  is
// accumulated in registers for the whole reverse pass as  dW2 += c * Delta2 * H1'  (a [64 x TB] x [TB x 64] product per
// stage point) -- grad is ONE shared vector per block, not the reference's per-trajectory (n+P)-long augmented state
// (src/interpolating_adjoint.jl:387-394).  Block partials are then summed in block order (deterministic).
//
// Reference functions replaced: sense functor src/interpolating_adjoint.jl:150-174, split_states :190-205,
// vecjacobian! with its AD back-ends src/derivative_wrappers.jl:256-267, :800-928 (ZygoteVJP on a Lux/Flux chain),
// ReverseLossCallback src/adjoint_common.jl:754-821; hand VJP: SURVEY.md App. C.
// Parameter layout (column-major flatten of [W1(64x2), b1, W2(64x64), b2, W3(2x64), b3], P = 4482): as the oracle.
#pragma once
#include <cuda_runtime.h>
#include <stdint.h>
#include <cuda_bf16.h>
#include "ode_tsit5.cuh"

namespace b200adj {

constexpr int MLP_H = 64, MLP_D = 2, MLP_TB = 32, MLP_THREADS = 256;
constexpr int MLP_P = MLP_H * MLP_D + MLP_H + MLP_H * MLP_H + MLP_H + MLP_D * MLP_H + MLP_D;   // 4482
constexpr int MLP_OW1 = 0, MLP_OB1 = MLP_H * MLP_D, MLP_OW2 = MLP_OB1 + MLP_H, MLP_OB2 = MLP_OW2 + MLP_H * MLP_H,
              MLP_OW3 = MLP_OB2 + MLP_H, MLP_OB3 = MLP_OW3 + MLP_D * MLP_H;

template <class T> struct MlpArgs {
    const T* u0; const T* p; T* ckpt; T* saved; const int32_t* save_of_step; int32_t* status;
    const T* dLdu; T* du0; T* partials; T* dp;     // partials [grid][P]
    int64_t N; int32_t S; double cost_a[4], cost_b[4]; uint32_t flags;
    float* kst;                                       // tensor-core path: forward stages k1..k7 per step, [S][7][2][N]
    Tsit5Tables tb;
    // hybrid neural ODE (test/Core5/HybridNODE.jl:20-24, PresetTimeCallback on a neural RHS): preset-time events on the dt grid,
    // event_of_step[n] = e when u <- ev_s[e] .* u + ev_c[e] fires at t_n (else -1); null = none.  CUDA-core kernels (F64 / F32).
    const int32_t* event_of_step; const double* ev_s; const double* ev_c;
};

template <class T> __device__ __forceinline__ T tanh_t(T x);
template <> __device__ __forceinline__ double tanh_t<double>(double x) { return tanh(x); }
template <> __device__ __forceinline__ float tanh_t<float>(float x) { return tanhf(x); }

// shared-memory image of one block
template <class T> struct MlpSmem {
    T W1[MLP_D][MLP_H];          // W1[j][i]
    T b1[MLP_H], b2[MLP_H];
    T W2F[MLP_H][MLP_H];         // W2F[j][i] = W2[i][j]   (k = input j, m = output i)   forward product
    T W2B[MLP_H][MLP_H];         // W2B[i][j] = W2[i][j]   (k = output i, m = input j)   transposed product
    T W3[MLP_H][MLP_D];          // W3[j][c]
    T b3[MLP_D];
    T H1[MLP_H][MLP_TB], H2[MLP_H][MLP_TB], D1[MLP_H][MLP_TB], D2[MLP_H][MLP_TB];
    T y[MLP_D][MLP_TB], F[MLP_D][MLP_TB], L[MLP_D][MLP_TB], JTL[MLP_D][MLP_TB];
    T lam[MLP_D][MLP_TB], uhi[MLP_D][MLP_TB], ulo[MLP_D][MLP_TB];
    T kf[7][MLP_D][MLP_TB], ka[7][MLP_D][MLP_TB];
};

template <class T>
__device__ __forceinline__ void mlp_load_params(MlpSmem<T>& s, const T* p) {
    for (int x = threadIdx.x; x < MLP_H * MLP_D; x += MLP_THREADS) { int j = x / MLP_H, i = x % MLP_H; s.W1[j][i] = p[MLP_OW1 + x]; }
    for (int x = threadIdx.x; x < MLP_H; x += MLP_THREADS) { s.b1[x] = p[MLP_OB1 + x]; s.b2[x] = p[MLP_OB2 + x]; }
    for (int x = threadIdx.x; x < MLP_H * MLP_H; x += MLP_THREADS) { int j = x / MLP_H, i = x % MLP_H; T w = p[MLP_OW2 + x]; s.W2F[j][i] = w; s.W2B[i][j] = w; }
    for (int x = threadIdx.x; x < MLP_H * MLP_D; x += MLP_THREADS) { int j = x / MLP_D, c = x % MLP_D; s.W3[j][c] = p[MLP_OW3 + x]; }
    if (threadIdx.x < MLP_D) s.b3[threadIdx.x] = p[MLP_OB3 + threadIdx.x];
}

// acc[4][2] = sum_k Wk[k][m0..m0+3] * X[k][b0..b0+1]   (64 x 64 x TB product, 4 x 2 register tile per thread)
template <class T>
__device__ __forceinline__ void mlp_gemm(const T (*Wk)[MLP_H], const T (*X)[MLP_TB], int m0, int b0, T acc[4][2]) {
#pragma unroll
    for (int r = 0; r < 4; r++) { acc[r][0] = 0; acc[r][1] = 0; }
#pragma unroll 8
    for (int k = 0; k < MLP_H; k++) {
        const T x0 = X[k][b0], x1 = X[k][b0 + 1];
#pragma unroll
        for (int r = 0; r < 4; r++) { const T w = Wk[k][m0 + r]; acc[r][0] = fma(w, x0, acc[r][0]); acc[r][1] = fma(w, x1, acc[r][1]); }
    }
}

// forward pass at s.y -> s.H1, s.H2, s.F  (ends with a barrier)
template <class T>
__device__ __forceinline__ void mlp_forward(MlpSmem<T>& s) {
    const int m0 = (threadIdx.x / 16) * 4, b0 = (threadIdx.x % 16) * 2;
    for (int x = threadIdx.x; x < MLP_H * MLP_TB; x += MLP_THREADS) {
        const int i = x / MLP_TB, b = x % MLP_TB;
        s.H1[i][b] = tanh_t<T>(fma(s.W1[0][i], s.y[0][b], fma(s.W1[1][i], s.y[1][b], s.b1[i])));
    }
    __syncthreads();
    T acc[4][2];
    mlp_gemm<T>(s.W2F, s.H1, m0, b0, acc);
#pragma unroll
    for (int r = 0; r < 4; r++) { s.H2[m0 + r][b0] = tanh_t<T>(acc[r][0] + s.b2[m0 + r]); s.H2[m0 + r][b0 + 1] = tanh_t<T>(acc[r][1] + s.b2[m0 + r]); }
    __syncthreads();
    if (threadIdx.x < MLP_D * MLP_TB) {
        const int c = threadIdx.x / MLP_TB, b = threadIdx.x % MLP_TB;
        T v = s.b3[c];
#pragma unroll 8
        for (int j = 0; j < MLP_H; j++) v = fma(s.W3[j][c], s.H2[j][b], v);
        s.F[c][b] = v;
    }
    __syncthreads();
}

// backward pass of cotangent s.L through the network evaluated by the last mlp_forward -> s.D2, s.D1, s.JTL = J' L
template <class T>
__device__ __forceinline__ void mlp_backward(MlpSmem<T>& s) {
    const int m0 = (threadIdx.x / 16) * 4, b0 = (threadIdx.x % 16) * 2;
    for (int x = threadIdx.x; x < MLP_H * MLP_TB; x += MLP_THREADS) {
        const int j = x / MLP_TB, b = x % MLP_TB;
        const T h = s.H2[j][b];
        s.D2[j][b] = fma(s.W3[j][0], s.L[0][b], s.W3[j][1] * s.L[1][b]) * (T(1) - h * h);
    }
    __syncthreads();
    T acc[4][2];
    mlp_gemm<T>(s.W2B, s.D2, m0, b0, acc);
#pragma unroll
    for (int r = 0; r < 4; r++) {
        const T h0 = s.H1[m0 + r][b0], h1 = s.H1[m0 + r][b0 + 1];
        s.D1[m0 + r][b0] = acc[r][0] * (T(1) - h0 * h0); s.D1[m0 + r][b0 + 1] = acc[r][1] * (T(1) - h1 * h1);
    }
    __syncthreads();
    if (threadIdx.x < MLP_D * MLP_TB) {
        const int c = threadIdx.x / MLP_TB, b = threadIdx.x % MLP_TB;
        T v = 0;
#pragma unroll 8
        for (int i = 0; i < MLP_H; i++) v = fma(s.W1[c][i], s.D1[i][b], v);
        s.JTL[c][b] = v;
    }
    __syncthreads();
}

// per-thread slice of the parameter gradient
template <class T> struct MlpGrad {
    T w2[4][4];      // dW2[i0..i0+3][j0..j0+3], i0 = (tid/16)*4, j0 = (tid%16)*4
    T a, b, c, d;    // tid < 64: db1[i], db2[i], dW1[i][0], dW1[i][1] ; 64 <= tid < 128: dW3[0][j], dW3[1][j] in a, b ; tid 128,129: db3[c] in a
};

// grad += c * F(y)' L  with the activations of the last forward/backward pair (s.y, s.L, s.H1, s.H2, s.D1, s.D2), members >= nvalid masked
template <class T>
__device__ __forceinline__ void mlp_accumulate(const MlpSmem<T>& s, MlpGrad<T>& g, T c, int nvalid) {
    const int i0 = (threadIdx.x / 16) * 4, j0 = (threadIdx.x % 16) * 4, t = threadIdx.x;
    for (int b = 0; b < nvalid; b++) {
        T d[4], h[4];
#pragma unroll
        for (int r = 0; r < 4; r++) { d[r] = c * s.D2[i0 + r][b]; h[r] = s.H1[j0 + r][b]; }
#pragma unroll
        for (int r = 0; r < 4; r++)
#pragma unroll
            for (int q = 0; q < 4; q++) g.w2[r][q] = fma(d[r], h[q], g.w2[r][q]);
    }
    if (t < MLP_H) {
        T s1 = 0, s2 = 0, w0 = 0, w1 = 0;
        for (int b = 0; b < nvalid; b++) { const T d1 = s.D1[t][b]; s1 += d1; s2 += s.D2[t][b]; w0 = fma(d1, s.y[0][b], w0); w1 = fma(d1, s.y[1][b], w1); }
        g.a = fma(c, s1, g.a); g.b = fma(c, s2, g.b); g.c = fma(c, w0, g.c); g.d = fma(c, w1, g.d);
    } else if (t < 2 * MLP_H) {
        const int j = t - MLP_H; T w0 = 0, w1 = 0;
        for (int b = 0; b < nvalid; b++) { const T h = s.H2[j][b]; w0 = fma(s.L[0][b], h, w0); w1 = fma(s.L[1][b], h, w1); }
        g.a = fma(c, w0, g.a); g.b = fma(c, w1, g.b);
    } else if (t < 2 * MLP_H + MLP_D) {
        const int cc = t - 2 * MLP_H; T s1 = 0;
        for (int b = 0; b < nvalid; b++) s1 += s.L[cc][b];
        g.a = fma(c, s1, g.a);
    }
}

template <class T>
__device__ __forceinline__ void mlp_store_grad(const MlpGrad<T>& g, T* out /*[P]*/) {
    const int i0 = (threadIdx.x / 16) * 4, j0 = (threadIdx.x % 16) * 4, t = threadIdx.x;
#pragma unroll
    for (int r = 0; r < 4; r++)
#pragma unroll
        for (int q = 0; q < 4; q++) out[MLP_OW2 + (j0 + q) * MLP_H + (i0 + r)] = g.w2[r][q];
    if (t < MLP_H) { out[MLP_OB1 + t] = g.a; out[MLP_OB2 + t] = g.b; out[MLP_OW1 + 0 * MLP_H + t] = g.c; out[MLP_OW1 + 1 * MLP_H + t] = g.d; }
    else if (t < 2 * MLP_H) { const int j = t - MLP_H; out[MLP_OW3 + j * MLP_D + 0] = g.a; out[MLP_OW3 + j * MLP_D + 1] = g.b; }
    else if (t < 2 * MLP_H + MLP_D) out[MLP_OB3 + (t - 2 * MLP_H)] = g.a;
}

// ---- forward ensemble solve ----
template <class T>
__global__ void __launch_bounds__(MLP_THREADS) mlp_forward_kernel(const __grid_constant__ MlpArgs<T> a) {
    extern __shared__ __align__(16) unsigned char smem_raw[];
    MlpSmem<T>& s = *reinterpret_cast<MlpSmem<T>*>(smem_raw);
    const int64_t N = a.N, base = (int64_t)blockIdx.x * MLP_TB;
    const int nvalid = (int)min((int64_t)MLP_TB, N - base);
    const int t = threadIdx.x, c = t / MLP_TB, b = t % MLP_TB;            // t < 64: (component, member) owner
    const bool own = t < MLP_D * MLP_TB, live = own && b < nvalid;
    const int64_t col = base + (b < nvalid ? b : nvalid - 1);
    mlp_load_params<T>(s, a.p);
    if (own) { s.ulo[c][b] = a.u0[(int64_t)c * N + col]; s.y[c][b] = s.ulo[c][b]; }
    __syncthreads();
    if (live) { a.ckpt[(int64_t)c * N + col] = s.ulo[c][b]; if (a.saved) { int ks = a.save_of_step[0]; if (ks >= 0) a.saved[((int64_t)ks * MLP_D + c) * N + col] = s.ulo[c][b]; } }
    mlp_forward<T>(s);
    if (own) s.kf[0][c][b] = s.F[c][b];
    __syncthreads();
    for (int n = 0; n < a.S; n++) {
#pragma unroll 1
        for (int st = 1; st <= 6; st++) {
            if (own) {
                double acc = (double)s.ulo[c][b];
                for (int j = 0; j < st; j++) acc = fma(a.tb.hA[st][j], (double)s.kf[j][c][b], acc);
                s.y[c][b] = (T)acc;
            }
            __syncthreads();
            mlp_forward<T>(s);
            if (own) { if (st < 6) s.kf[st][c][b] = s.F[c][b]; else { s.ulo[c][b] = s.y[c][b]; s.kf[0][c][b] = s.F[c][b]; } }
            __syncthreads();
        }
        if (a.event_of_step) {
            // preset-time event at t_{n+1}: the checkpoint and a coinciding save point record the POST-event state, the first
            // stage of the next step is re-evaluated from it (same convention as tsit5_forward_kernel<..., EV>)
            const int e = a.event_of_step[n + 1];
            if (e >= 0 && n + 1 < a.S) {
                if (own) { s.ulo[c][b] = (T)(a.ev_s[e * MLP_D + c] * (double)s.ulo[c][b] + a.ev_c[e * MLP_D + c]); s.y[c][b] = s.ulo[c][b]; }
                __syncthreads();
                mlp_forward<T>(s);
                if (own) s.kf[0][c][b] = s.F[c][b];
                __syncthreads();
            }
        }
        if (live) {
            a.ckpt[((int64_t)(n + 1) * MLP_D + c) * N + col] = s.ulo[c][b];
            if (a.saved) { int ks = a.save_of_step[n + 1]; if (ks >= 0) a.saved[((int64_t)ks * MLP_D + c) * N + col] = s.ulo[c][b]; }
        }
    }
    if (live && c == 0 && a.status) a.status[col] = (isfinite((double)s.ulo[0][b]) && isfinite((double)s.ulo[1][b])) ? 0 : 1;
}

// ---- fused reverse pass.  GAUSS = false: InterpolatingAdjoint (mu integrated with the adjoint tableau); GAUSS = true:
// GaussAdjoint (the reference's default once length(u0) + length(p) > 100, src/concrete_solve.jl:291-316): state lambda only,
// dp += (h/2) w_g F(y_g)' lam_g at the three Gauss-Legendre nodes of every step, lam_g from the adjoint step's own dense
// output and y_g from the forward dense output (src/gauss_adjoint.jl:745-759) ----
template <class T, int COST, bool GAUSS>
__global__ void __launch_bounds__(MLP_THREADS) mlp_reverse_kernel(const __grid_constant__ MlpArgs<T> a) {
    extern __shared__ __align__(16) unsigned char smem_raw[];
    MlpSmem<T>& s = *reinterpret_cast<MlpSmem<T>*>(smem_raw);
    const int64_t N = a.N, base = (int64_t)blockIdx.x * MLP_TB;
    const int nvalid = (int)min((int64_t)MLP_TB, N - base);
    const int t = threadIdx.x, c = t / MLP_TB, b = t % MLP_TB;
    const bool own = t < MLP_D * MLP_TB, live = own && b < nvalid;
    const int64_t col = base + (b < nvalid ? b : nvalid - 1);
    const Tsit5Tables& tb = a.tb;
    mlp_load_params<T>(s, a.p);
    MlpGrad<T> g;
#pragma unroll
    for (int r = 0; r < 4; r++)
#pragma unroll
        for (int q = 0; q < 4; q++) g.w2[r][q] = 0;
    g.a = g.b = g.c = g.d = 0;
    auto cotangent = [&](int ks, const T (*yy)[MLP_TB]) {      // lam += dgdu at save index ks (owner threads)
        if (own) {
            if (COST == COST_EXPLICIT) s.lam[c][b] += a.dLdu[((int64_t)ks * MLP_D + c) * N + col];
            else s.lam[c][b] += (T)(a.cost_a[c] * (double)yy[c][b] + a.cost_b[c]);
        }
    };
    if (own) { s.lam[c][b] = 0; s.uhi[c][b] = a.ckpt[((int64_t)a.S * MLP_D + c) * N + col]; s.y[c][b] = s.uhi[c][b]; }
    __syncthreads();
    { int ks = a.save_of_step[a.S]; if (ks >= 0) cotangent(ks, s.uhi); }
    mlp_forward<T>(s);                                          // f(u_S) = forward k7 of the last step
    if (own) s.kf[6][c][b] = s.F[c][b];
    __syncthreads();
    bool need_left = false;     // the step above ended with an event at t_{n+1}: its right end is the LEFT limit, not the checkpoint
    for (int n = a.S - 1; n >= 0; n--) {
        if (own) { s.ulo[c][b] = a.ckpt[((int64_t)n * MLP_D + c) * N + col]; s.y[c][b] = s.ulo[c][b]; }
        __syncthreads();
        // ---- forward stage recompute k1..k6 on [t_n, t_{n+1}] ----
        mlp_forward<T>(s);
        if (own) s.kf[0][c][b] = s.F[c][b];
        __syncthreads();
#pragma unroll 1
        for (int st = 1; st <= 5; st++) {
            if (own) {
                double acc = (double)s.ulo[c][b];
                for (int j = 0; j < st; j++) acc = fma(tb.hA[st][j], (double)s.kf[j][c][b], acc);
                s.y[c][b] = (T)acc;
            }
            __syncthreads();
            mlp_forward<T>(s);
            if (own) s.kf[st][c][b] = s.F[c][b];
            __syncthreads();
        }
        if (need_left) {
            // event at t_{n+1}: the adjoint step starts from the pre-event end state of this forward step, u- = u_n + h sum b_j k_j,
            // and the dense output needs k7 = f(u-) (the checkpoint above holds the post-event state)
            if (own) {
                double acc = (double)s.ulo[c][b];
                for (int j = 0; j < 6; j++) acc = fma(tb.hA[6][j], (double)s.kf[j][c][b], acc);
                s.uhi[c][b] = (T)acc; s.y[c][b] = (T)acc;
            }
            __syncthreads();
            mlp_forward<T>(s);
            if (own) s.kf[6][c][b] = s.F[c][b];
            __syncthreads();
            need_left = false;
        }
        // ---- adjoint stages 0..5 (b7 = 0: the 7th stage carries no mu weight; GaussAdjoint needs its derivative for the
        //      dense output of the adjoint step, so it runs stage 6 as well) ----
#pragma unroll 1
        for (int st = 0; st <= (GAUSS ? 6 : 5); st++) {
            if (own) {
                double l = (double)s.lam[c][b];
                for (int j = 0; j < st && j < 6; j++) l = fma(tb.hA[st][j], (double)s.ka[j][c][b], l);
                s.L[c][b] = (T)l;
                double yv;
                if (st == 0) yv = (double)s.uhi[c][b];
                else if (st >= 5) yv = (double)s.ulo[c][b];
                else { yv = (double)s.ulo[c][b]; for (int j = 0; j < 7; j++) yv = fma(tb.hBst[st - 1][j], (double)s.kf[j][c][b], yv); }
                s.y[c][b] = (T)yv;
            }
            __syncthreads();
            mlp_forward<T>(s);
            mlp_backward<T>(s);
            if (own) s.ka[st][c][b] = s.JTL[c][b];
            if (!GAUSS) mlp_accumulate<T>(s, g, (T)tb.hA[6][st], nvalid);
            __syncthreads();
        }
        if (GAUSS) {
#pragma unroll 1
            for (int gq = 0; gq < 3; gq++) {
                if (own) {
                    double l = (double)s.lam[c][b], yv = (double)s.ulo[c][b];
                    for (int j = 0; j < 7; j++) { l = fma(tb.hBq[gq][j], (double)s.ka[j][c][b], l); yv = fma(tb.hBq[2 - gq][j], (double)s.kf[j][c][b], yv); }
                    s.L[c][b] = (T)l; s.y[c][b] = (T)yv;
                }
                __syncthreads();
                mlp_forward<T>(s);
                mlp_backward<T>(s);
                mlp_accumulate<T>(s, g, (T)tb.hGW[gq], nvalid);
                __syncthreads();
            }
        }
        // lambda(t_n) = lam + sum_j h b_j ka_j ; jump at t_n ; shift
        if (own) {
            double l = (double)s.lam[c][b];
            for (int j = 0; j < 6; j++) l = fma(tb.hA[6][j], (double)s.ka[j][c][b], l);
            s.lam[c][b] = (T)l;
        }
        { const int ks = a.save_of_step[n]; if (ks >= 0 && !((a.flags & KF_NO_START) && n == 0)) cotangent(ks, s.ulo); }
        if (own) { s.uhi[c][b] = s.ulo[c][b]; s.kf[6][c][b] = s.kf[0][c][b]; }
        if (a.event_of_step) {
            // reverse affect of u+ = s .* u- + c at t_n, after the loss jump of the same time: lam- = s .* lam+
            const int e = a.event_of_step[n];
            if (e >= 0 && n > 0) { if (own) s.lam[c][b] = (T)(a.ev_s[e * MLP_D + c] * (double)s.lam[c][b]); need_left = true; }
        }
        __syncthreads();
    }
    if (live) a.du0[(int64_t)c * N + col] = s.lam[c][b];
    mlp_store_grad<T>(g, a.partials + (int64_t)blockIdx.x * MLP_P);
}

// dp[q] = sum over blocks (in block order) of partials[blk][q]
template <class T>
__global__ void mlp_reduce_kernel(const T* partials, T* dp, int nblocks) {
    const int q = blockIdx.x * blockDim.x + threadIdx.x;
    if (q >= MLP_P) return;
    double acc = 0;                                    // fp64 accumulation of the block partials in either precision
    for (int k = 0; k < nblocks; k++) acc += (double)partials[(int64_t)k * MLP_P + q];
    dp[q] = (T)acc;
}

}  // namespace b200adj
