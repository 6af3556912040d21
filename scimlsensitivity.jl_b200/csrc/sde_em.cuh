// sde_em.cuh -- SDE ensemble kernels: forward EM / EulerHeun and the BacksolveAdjoint / InterpolatingAdjoint reverse pass,
// for diagonal noise (g .* dW) and for general noise (G dW, G of size D x M).
// One member per thread, SoA [step][dim][member].  Wiener increments come from a Philox4x32-10 counter keyed by
// (seed, global member index, step) so the reverse pass REGENERATES them instead of reading a stored noise grid
// (the reference stores sol.W and integrates against reverse(W), src/backsolve_adjoint.jl:395-411); a stored-noise
// mode is kept for parity tests and reference-style NoiseGrid inputs.
//
// Reference functions replaced:  SDEAdjointProblem src/backsolve_adjoint.jl:274-419 (state z=[lam; mu; y], drift
// functor on f or on the Ito-transformed drift :327-345, diffusion functor noiseterm=true :347-357), sense functor
// arithmetic :32-61, noise layouts split_states :92-117, jacNoise! src/derivative_wrappers.jl:1165-1258,
// StochasticTransformedFunction src/sde_tools.jl:29-66, checkpoint reset :523-546, ReverseLossCallback
// src/adjoint_common.jl:754-821; upstream EM / EulerHeun steps (SURVEY.md App. B).
#pragma once
#include <cuda_runtime.h>
#include <stdint.h>
#include "families.cuh"
#include "ode_tsit5.cuh"

namespace b200adj {

struct SdeFwdArgs {
    const double* u0; const double* p; double* ckpt; double* saved; const int32_t* save_of_step; int32_t* status;
    const double* noise_in;   // [S][M][N] or null (Philox)
    double* noise_out;        // [S][M][N] or null
    int64_t N; int32_t S; double h; uint64_t seed; int64_t traj_offset;
};
struct SdeRevArgs {
    const double* ckpt; const double* p; const double* dLdu; const int32_t* save_of_step;
    double* du0; double* dp_members; double* partials; double* dp; unsigned int* ticket;
    const double* noise;      // [S][M][N] or null (regenerate)
    int64_t N; int32_t S; double h; double cost_a[4], cost_b[4]; uint32_t flags; uint64_t seed; int64_t traj_offset;
};
struct SdeNoiseArgs { double* out; int64_t N; int32_t S; double h; uint64_t seed; int64_t traj_offset; int32_t m; };

// ---- Philox4x32-10 (Salmon et al. 2011) ----
__device__ __forceinline__ void philox4x32_10(uint32_t c0, uint32_t c1, uint32_t c2, uint32_t c3, uint32_t k0, uint32_t k1, uint32_t* out) {
#pragma unroll
    for (int r = 0; r < 10; r++) {
        const uint32_t hi0 = __umulhi(0xD2511F53u, c0), lo0 = 0xD2511F53u * c0;
        const uint32_t hi1 = __umulhi(0xCD9E8D57u, c2), lo1 = 0xCD9E8D57u * c2;
        const uint32_t n0 = hi1 ^ c1 ^ k0, n1 = lo1, n2 = hi0 ^ c3 ^ k1, n3 = lo0;
        c0 = n0; c1 = n1; c2 = n2; c3 = n3;
        k0 += 0x9E3779B9u; k1 += 0xBB67AE85u;
    }
    out[0] = c0; out[1] = c1; out[2] = c2; out[3] = c3;
}
// two N(0,1) doubles for (member, step, pair) by Box-Muller on two 53-bit uniforms in (0,1)
__device__ __forceinline__ void normal_pair(uint64_t seed, uint64_t member, uint32_t step, uint32_t pair, double* z0, double* z1) {
    uint32_t r[4];
    philox4x32_10((uint32_t)member, (uint32_t)(member >> 32), step, pair, (uint32_t)seed, (uint32_t)(seed >> 32), r);
    const uint64_t a = ((uint64_t)r[0] << 21) ^ (uint64_t)(r[1] >> 11);
    const uint64_t b = ((uint64_t)r[2] << 21) ^ (uint64_t)(r[3] >> 11);
    const double u1 = ((double)a + 0.5) * 1.1102230246251565e-16;   // 2^-53
    const double u2 = ((double)b + 0.5) * 1.1102230246251565e-16;
    const double rad = sqrt(-2.0 * log(u1));
    double s, c;
    sincospi(2.0 * u2, &s, &c);
    *z0 = rad * c; *z1 = rad * s;
}
template <int M>
__device__ __forceinline__ void wiener_increment(uint64_t seed, uint64_t member, uint32_t step, double sqrth, double* dW) {
#pragma unroll
    for (int q = 0; q < (M + 1) / 2; q++) {
        double z0, z1;
        normal_pair(seed, member, step, (uint32_t)q, &z0, &z1);
        dW[2 * q] = sqrth * z0;
        if (2 * q + 1 < M) dW[2 * q + 1] = sqrth * z1;
    }
}

template <int UNUSED = 0>
__global__ void sde_noise_kernel(SdeNoiseArgs a) {
    const int64_t t = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (t >= (int64_t)a.S * a.N) return;
    const int64_t n = t / a.N, i = t % a.N;
    const double sq = sqrt(a.h);
    for (int q = 0; q < (a.m + 1) / 2; q++) {
        double z0, z1;
        normal_pair(a.seed, (uint64_t)(a.traj_offset + i), (uint32_t)n, (uint32_t)q, &z0, &z1);
        a.out[(n * a.m + 2 * q) * a.N + i] = sq * z0;
        if (2 * q + 1 < a.m) a.out[(n * a.m + 2 * q + 1) * a.N + i] = sq * z1;
    }
}

// The two noise shapes of an SDE family.  Diagonal (SdeLotkaVolterra): g(u, p, g) gives the diffusion of each component,
// one Wiener process per state (M == D), and the noise enters as g .* w.  General (a struct with g_apply): G(u, p) is D x M
// and the family supplies only its contractions with the increments w[M] -- the noise enters linearly, so the kernels never
// form the matrix the reference builds and multiplies by dW (src/derivative_wrappers.jl:1197-1258):
//   g_apply(u, p, w, out)            out = G w
//   gvjp_u_apply(u, p, l, w, dl)     dl = sum_j w_j (dG[:, j]/du)' l
//   gvjp_p_apply(u, p, l, w, dg)     dg = sum_j w_j (dG[:, j]/dp)' l        (the same name and meaning in both shapes)
// Each helper below has one form per shape; the diagonal forms are the expressions the kernels had before the general
// shape existed.
template <class Fam, class = void> struct SdeGeneralNoise { static constexpr bool value = false; };
template <class Fam> struct SdeGeneralNoise<Fam, decltype(void(&Fam::template g_apply<double>))> { static constexpr bool value = true; };

// the diffusion at (u, p) in the family's form: g (diagonal) or G w (general)
template <class Fam>
__device__ __forceinline__ void sde_diffusion(const double* u, const double* p, const double* w, double* g) {
    if constexpr (SdeGeneralNoise<Fam>::value) Fam::g_apply(u, p, w, g);
    else Fam::g(u, p, g);
}
// its noise term in component j: g_j w_j or (G w)_j
template <class Fam>
__device__ __forceinline__ double sde_noise(const double* g, const double* w, int j) {
    if constexpr (SdeGeneralNoise<Fam>::value) return g[j];
    else return g[j] * w[j];
}
// EulerHeun's averaged noise term from the diffusions at u and at the predictor
template <class Fam>
__device__ __forceinline__ double sde_noise_avg(const double* g, const double* gb, const double* w, int j) {
    if constexpr (SdeGeneralNoise<Fam>::value) return 0.5 * (g[j] + gb[j]);
    else return 0.5 * (g[j] + gb[j]) * w[j];
}
// the u-part of the diffusion VJP in the family's form: l .* dg/du (diagonal) or sum_j w_j (dG[:, j]/du)' l (general);
// sde_noise turns either into the reverse diffusion increment
template <class Fam>
__device__ __forceinline__ void sde_diffusion_vjp_u(const double* u, const double* p, const double* l, const double* w, double* dl) {
    if constexpr (SdeGeneralNoise<Fam>::value) Fam::gvjp_u_apply(u, p, l, w, dl);
    else Fam::gvjp_u(u, p, l, dl);
}

template <class Fam, bool EULER_HEUN, bool SHARED_P>
__global__ void __launch_bounds__(512) sde_forward_kernel(SdeFwdArgs a) {
    const int BLOCK = (int)blockDim.x;
    constexpr int D = Fam::D, P = Fam::P, M = Fam::M;
    static_assert(SdeGeneralNoise<Fam>::value || M == D, "diagonal noise: one Wiener process per state");
    const int64_t gi = (int64_t)blockIdx.x * BLOCK + threadIdx.x;
    const bool active = gi < a.N;
    const int64_t i = active ? gi : a.N - 1;
    const int64_t N = a.N, stride = (int64_t)D * N;
    double p[P];
#pragma unroll
    for (int q = 0; q < P; q++) p[q] = SHARED_P ? __ldg(a.p + q) : __ldg(a.p + (int64_t)q * N + i);
    double u[D], f[D], g[D], dW[M];
    load_state<D>(a.u0, N, i, u);
    if (active) {
        store_state<D>(a.ckpt, N, i, u);
        if (a.saved) { int ks = a.save_of_step[0]; if (ks >= 0) store_state<D>(a.saved + (int64_t)ks * stride, N, i, u); }
    }
    const double h = a.h, sq = sqrt(a.h);
    for (int n = 0; n < a.S; n++) {
        if (a.noise_in) load_state<M>(a.noise_in + (int64_t)n * M * N, N, i, dW);
        else wiener_increment<M>(a.seed, (uint64_t)(a.traj_offset + i), (uint32_t)n, sq, dW);
        if (a.noise_out && active) store_state<M>(a.noise_out + (int64_t)n * M * N, N, i, dW);
        Fam::f(u, p, f); sde_diffusion<Fam>(u, p, dW, g);
        if (!EULER_HEUN) {
#pragma unroll
            for (int j = 0; j < D; j++) u[j] = u[j] + h * f[j] + sde_noise<Fam>(g, dW, j);
        } else {
            double ub[D], fb[D], gb[D];
#pragma unroll
            for (int j = 0; j < D; j++) ub[j] = u[j] + h * f[j] + sde_noise<Fam>(g, dW, j);
            Fam::f(ub, p, fb); sde_diffusion<Fam>(ub, p, dW, gb);
#pragma unroll
            for (int j = 0; j < D; j++) u[j] = u[j] + 0.5 * h * (f[j] + fb[j]) + sde_noise_avg<Fam>(g, gb, dW, j);
        }
        if (active) {
            store_state<D>(a.ckpt + (int64_t)(n + 1) * stride, N, i, u);
            if (a.saved) { int ks = a.save_of_step[n + 1]; if (ks >= 0) store_state<D>(a.saved + (int64_t)ks * stride, N, i, u); }
        }
    }
    if (active && a.status) {
        bool ok = true;
#pragma unroll
        for (int j = 0; j < D; j++) ok = ok && isfinite(u[j]);
        a.status[i] = ok ? 0 : 1;
    }
}

// drift a(z) and diffusion increment b(z; w) of the augmented reverse SDE, z = [lam; mu; y]
template <class Fam, int D, int P>
__device__ __forceinline__ void sde_adj_terms(const double* lam, const double* y, const double* p, const double* w,
                                              double* al, double* am, double* ay, double* bl, double* bm, double* by) {
    double g[D], gl[D];
    Fam::vjp_u(y, p, lam, al); Fam::vjp_p(y, p, lam, am); Fam::f(y, p, ay);
    sde_diffusion<Fam>(y, p, w, g); sde_diffusion_vjp_u<Fam>(y, p, lam, w, gl); Fam::gvjp_p_apply(y, p, lam, w, bm);
#pragma unroll
    for (int j = 0; j < D; j++) { al[j] = -al[j]; bl[j] = -sde_noise<Fam>(gl, w, j); by[j] = sde_noise<Fam>(g, w, j); }
#pragma unroll
    for (int q = 0; q < P; q++) { am[q] = -am[q]; bm[q] = -bm[q]; }
}

// INTERP = false: BacksolveAdjoint, z = [lam; mu; y] (y integrated backwards, reset at checkpoints).
// INTERP = true : InterpolatingAdjoint (src/interpolating_adjoint.jl:453-613), z = [lam; mu]; y(t) is read from the saved
//                 forward solution at every grid point (the reverse solve steps on the forward grid) and the drift is the
//                 problem's f without the Ito transformation (the caller instantiates Fam with ITO = false).
template <class Fam, bool EULER_HEUN, bool SHARED_P, int COST, bool INTERP>
__global__ void __launch_bounds__(512) sde_backsolve_kernel(SdeRevArgs a) {
    const int BLOCK = (int)blockDim.x;
    constexpr int D = Fam::D, P = Fam::P, M = Fam::M;
    const int64_t gi = (int64_t)blockIdx.x * BLOCK + threadIdx.x;
    const bool active = gi < a.N;
    const int64_t i = active ? gi : a.N - 1;
    const int64_t N = a.N, stride = (int64_t)D * N;
    double p[P];
#pragma unroll
    for (int q = 0; q < P; q++) p[q] = SHARED_P ? __ldg(a.p + q) : __ldg(a.p + (int64_t)q * N + i);
    double lam[D], mu[P], y[D];
#pragma unroll
    for (int j = 0; j < D; j++) lam[j] = 0.0;
#pragma unroll
    for (int q = 0; q < P; q++) mu[q] = 0.0;
    load_state<D>(a.ckpt + (int64_t)a.S * stride, N, i, y);
    const bool ckpt_on = !(a.flags & KF_NO_CHECKPOINTING), every = (a.flags & KF_CKPT_EVERY_STEP);
    const double h = a.h, sq = sqrt(a.h);
    for (int n = a.S; n >= 0; n--) {
        // callbacks at grid point n: checkpoint reset, then the loss jump
        const int ks = a.save_of_step[n];
        if (INTERP || (ckpt_on && (every || ks >= 0))) load_state<D>(a.ckpt + (int64_t)n * stride, N, i, y);
        // no_start skips the jump of the first save time for every sensealg but Backsolve (src/adjoint_common.jl:761)
        if (ks >= 0 && !(INTERP && (a.flags & KF_NO_START) && ks == 0)) {
            if (COST == COST_EXPLICIT) {
#pragma unroll
                for (int j = 0; j < D; j++) lam[j] += __ldg(a.dLdu + (int64_t)ks * stride + (int64_t)j * N + i);
            } else {
#pragma unroll
                for (int j = 0; j < D; j++) lam[j] += fma(a.cost_a[j], y[j], a.cost_b[j]);
            }
        }
        if (n == 0) break;
        // reverse step n -> n-1 with dt = -h and dW_rev = W(t_{n-1}) - W(t_n) = -dW_{n-1}
        double w[M];
        if (a.noise) load_state<M>(a.noise + (int64_t)(n - 1) * M * N, N, i, w);
        else wiener_increment<M>(a.seed, (uint64_t)(a.traj_offset + i), (uint32_t)(n - 1), sq, w);
#pragma unroll
        for (int j = 0; j < M; j++) w[j] = -w[j];
        double al[D], am[P], ay[D], bl[D], bm[P], by[D];
        sde_adj_terms<Fam, D, P>(lam, y, p, w, al, am, ay, bl, bm, by);
        if (!EULER_HEUN) {
#pragma unroll
            for (int j = 0; j < D; j++) { lam[j] = lam[j] - h * al[j] + bl[j]; y[j] = y[j] - h * ay[j] + by[j]; }
#pragma unroll
            for (int q = 0; q < P; q++) mu[q] = mu[q] - h * am[q] + bm[q];
        } else {
            double l2[D], y2[D], al2[D], am2[P], ay2[D], bl2[D], bm2[P], by2[D];
#pragma unroll
            for (int j = 0; j < D; j++) { l2[j] = lam[j] - h * al[j] + bl[j]; y2[j] = y[j] - h * ay[j] + by[j]; }
            if (INTERP) load_state<D>(a.ckpt + (int64_t)(n - 1) * stride, N, i, y2);      // y(t_{n-1}) = sol(t_{n-1})
            sde_adj_terms<Fam, D, P>(l2, y2, p, w, al2, am2, ay2, bl2, bm2, by2);
#pragma unroll
            for (int j = 0; j < D; j++) {
                lam[j] = lam[j] - 0.5 * h * (al[j] + al2[j]) + 0.5 * (bl[j] + bl2[j]);
                y[j] = y[j] - 0.5 * h * (ay[j] + ay2[j]) + 0.5 * (by[j] + by2[j]);
            }
#pragma unroll
            for (int q = 0; q < P; q++) mu[q] = mu[q] - 0.5 * h * (am[q] + am2[q]) + 0.5 * (bm[q] + bm2[q]);
        }
    }
    if (active) store_state<D>(a.du0, N, i, lam);
    store_dp<P, SHARED_P>(mu, active, i, N, a.dp_members, a.partials, a.dp, a.ticket);
}

}  // namespace b200adj
