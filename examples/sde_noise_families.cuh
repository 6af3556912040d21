// sde_noise_families.cuh -- USER general-noise SDE families for libb200adj.so (not part of the library):
// du = f(u, p) dt + G(u, p) dW with G of size D x M, in the shape csrc/family_plugin.inc describes for
// B200ADJ_FAMILY_SDE_GENERAL.  The family supplies G only through its contractions with the increments w[M]:
//   g_apply(u, p, w, out)          out = G w
//   gvjp_u_apply(u, p, l, w, dl)   dl  = sum_j w_j (dG[:, j]/du)' l
//   gvjp_p_apply(u, p, l, w, dg)   dg  = sum_j w_j (dG[:, j]/dp)' l
// The drift f is the problem's own (Stratonovich for EulerHeun); these families run on EM / EulerHeun with BacksolveAdjoint
// or InterpolatingAdjoint, except EM + BacksolveAdjoint.
// Build + register:  python -m scimlsensitivity_jl_b200.family_plugin examples/sde_noise_families.cuh SdeRoessler sde_roessler --sde --general-noise
#pragma once

// Non-diagonal noise of the reference's test/SDE2/sde_nondiag_stratonovich.jl:28-80 (Roessler, SIAM J. Numer. Anal. 48,
// 922-952, d = m = 2):  f = A u,  G[:, j] = B u  for both j,  A = [p0 p1; p1 p0],  B = [p2 p3; p3 p2].  A and B commute, so the
// Stratonovich solution is u(t) = expm(A t + B (W1(t) + W2(t))) u0.                                   D = 2, P = 4, M = 2
struct SdeRoessler {
    static constexpr int D = 2, P = 4, M = 2;
    template <class T> __device__ __forceinline__ static void f(const T* u, const T* p, T* du) {
        du[0] = p[0] * u[0] + p[1] * u[1];
        du[1] = p[1] * u[0] + p[0] * u[1];
    }
    template <class T> __device__ __forceinline__ static void vjp_u(const T* u, const T* p, const T* l, T* dl) {
        dl[0] = p[0] * l[0] + p[1] * l[1];
        dl[1] = p[1] * l[0] + p[0] * l[1];
    }
    template <class T> __device__ __forceinline__ static void vjp_p(const T* u, const T* p, const T* l, T* dg) {
        dg[0] = u[0] * l[0] + u[1] * l[1]; dg[1] = u[1] * l[0] + u[0] * l[1]; dg[2] = 0; dg[3] = 0;
    }
    // G w = (B u) (w0 + w1)
    template <class T> __device__ __forceinline__ static void g_apply(const T* u, const T* p, const T* w, T* out) {
        const T s = w[0] + w[1];
        out[0] = (p[2] * u[0] + p[3] * u[1]) * s;
        out[1] = (p[3] * u[0] + p[2] * u[1]) * s;
    }
    template <class T> __device__ __forceinline__ static void gvjp_u_apply(const T* u, const T* p, const T* l, const T* w, T* dl) {
        const T s = w[0] + w[1];
        dl[0] = (p[2] * l[0] + p[3] * l[1]) * s;
        dl[1] = (p[3] * l[0] + p[2] * l[1]) * s;
    }
    template <class T> __device__ __forceinline__ static void gvjp_p_apply(const T* u, const T* p, const T* l, const T* w, T* dg) {
        const T s = w[0] + w[1];
        dg[0] = 0; dg[1] = 0;
        dg[2] = (u[0] * l[0] + u[1] * l[1]) * s;
        dg[3] = (u[1] * l[0] + u[0] * l[1]) * s;
    }
};

// Diagonal noise that mixes (test/SDE2/sde_nondiag_stratonovich.jl:290-322, noisemixing = true):  the drift of SdeRoessler,
// G = diag(c, c) with c = p2 u0 + p3 u1, so g_1 depends on u_2.                                       D = 2, P = 4, M = 2
struct SdeMixing {
    static constexpr int D = 2, P = 4, M = 2;
    template <class T> __device__ __forceinline__ static void f(const T* u, const T* p, T* du) { SdeRoessler::f(u, p, du); }
    template <class T> __device__ __forceinline__ static void vjp_u(const T* u, const T* p, const T* l, T* dl) { SdeRoessler::vjp_u(u, p, l, dl); }
    template <class T> __device__ __forceinline__ static void vjp_p(const T* u, const T* p, const T* l, T* dg) { SdeRoessler::vjp_p(u, p, l, dg); }
    template <class T> __device__ __forceinline__ static void g_apply(const T* u, const T* p, const T* w, T* out) {
        const T c = p[2] * u[0] + p[3] * u[1];
        out[0] = c * w[0]; out[1] = c * w[1];
    }
    // l' G w = c (l0 w0 + l1 w1)
    template <class T> __device__ __forceinline__ static void gvjp_u_apply(const T* u, const T* p, const T* l, const T* w, T* dl) {
        const T s = l[0] * w[0] + l[1] * w[1];
        dl[0] = p[2] * s; dl[1] = p[3] * s;
    }
    template <class T> __device__ __forceinline__ static void gvjp_p_apply(const T* u, const T* p, const T* l, const T* w, T* dg) {
        const T s = l[0] * w[0] + l[1] * w[1];
        dg[0] = 0; dg[1] = 0; dg[2] = u[0] * s; dg[3] = u[1] * s;
    }
};

// Non-diagonal additive noise (test/SDE2/sde_nondiag_stratonovich.jl:793-822):  f = -u,  G = [K_R 0; K_I 0],  p = [K_R, K_I].
//                                                                                                      D = 2, P = 2, M = 2
struct SdeAdditive {
    static constexpr int D = 2, P = 2, M = 2;
    template <class T> __device__ __forceinline__ static void f(const T* u, const T* p, T* du) { du[0] = -u[0]; du[1] = -u[1]; }
    template <class T> __device__ __forceinline__ static void vjp_u(const T* u, const T* p, const T* l, T* dl) { dl[0] = -l[0]; dl[1] = -l[1]; }
    template <class T> __device__ __forceinline__ static void vjp_p(const T* u, const T* p, const T* l, T* dg) { dg[0] = 0; dg[1] = 0; }
    template <class T> __device__ __forceinline__ static void g_apply(const T* u, const T* p, const T* w, T* out) {
        out[0] = p[0] * w[0]; out[1] = p[1] * w[0];
    }
    template <class T> __device__ __forceinline__ static void gvjp_u_apply(const T* u, const T* p, const T* l, const T* w, T* dl) { dl[0] = 0; dl[1] = 0; }
    template <class T> __device__ __forceinline__ static void gvjp_p_apply(const T* u, const T* p, const T* l, const T* w, T* dg) {
        dg[0] = l[0] * w[0]; dg[1] = l[1] * w[0];
    }
};

// Non-square diffusion (test/SDE2/sde_nondiag_stratonovich.jl:863-885):  f = p0 u,  G = [p1 u0 0; 0 p1 u1; 0 0].  Component i
// < 2 is u0_i exp(p0 t + p1 W_i(t)) (Stratonovich), component 2 is u0_2 exp(p0 t).                 D = 3, P = 2, M = 2
struct SdeNonSquare {
    static constexpr int D = 3, P = 2, M = 2;
    template <class T> __device__ __forceinline__ static void f(const T* u, const T* p, T* du) { du[0] = p[0] * u[0]; du[1] = p[0] * u[1]; du[2] = p[0] * u[2]; }
    template <class T> __device__ __forceinline__ static void vjp_u(const T* u, const T* p, const T* l, T* dl) { dl[0] = p[0] * l[0]; dl[1] = p[0] * l[1]; dl[2] = p[0] * l[2]; }
    template <class T> __device__ __forceinline__ static void vjp_p(const T* u, const T* p, const T* l, T* dg) {
        dg[0] = u[0] * l[0] + u[1] * l[1] + u[2] * l[2]; dg[1] = 0;
    }
    template <class T> __device__ __forceinline__ static void g_apply(const T* u, const T* p, const T* w, T* out) {
        out[0] = p[1] * u[0] * w[0]; out[1] = p[1] * u[1] * w[1]; out[2] = 0;
    }
    template <class T> __device__ __forceinline__ static void gvjp_u_apply(const T* u, const T* p, const T* l, const T* w, T* dl) {
        dl[0] = p[1] * l[0] * w[0]; dl[1] = p[1] * l[1] * w[1]; dl[2] = 0;
    }
    template <class T> __device__ __forceinline__ static void gvjp_p_apply(const T* u, const T* p, const T* l, const T* w, T* dg) {
        dg[0] = 0; dg[1] = u[0] * l[0] * w[0] + u[1] * l[1] * w[1];
    }
};

// Scalar noise (test/SDE1/sde_scalar_stratonovich.jl:27-47): one Wiener process shared by both states,  f = p0 u,
// G[:, 0] = p1 u; the Stratonovich solution is u0 exp(p0 t + p1 W(t)).                               D = 2, P = 2, M = 1
struct SdeScalarLinear {
    static constexpr int D = 2, P = 2, M = 1;
    template <class T> __device__ __forceinline__ static void f(const T* u, const T* p, T* du) { du[0] = p[0] * u[0]; du[1] = p[0] * u[1]; }
    template <class T> __device__ __forceinline__ static void vjp_u(const T* u, const T* p, const T* l, T* dl) { dl[0] = p[0] * l[0]; dl[1] = p[0] * l[1]; }
    template <class T> __device__ __forceinline__ static void vjp_p(const T* u, const T* p, const T* l, T* dg) { dg[0] = u[0] * l[0] + u[1] * l[1]; dg[1] = 0; }
    template <class T> __device__ __forceinline__ static void g_apply(const T* u, const T* p, const T* w, T* out) {
        out[0] = p[1] * u[0] * w[0]; out[1] = p[1] * u[1] * w[0];
    }
    template <class T> __device__ __forceinline__ static void gvjp_u_apply(const T* u, const T* p, const T* l, const T* w, T* dl) {
        dl[0] = p[1] * l[0] * w[0]; dl[1] = p[1] * l[1] * w[0];
    }
    template <class T> __device__ __forceinline__ static void gvjp_p_apply(const T* u, const T* p, const T* l, const T* w, T* dg) {
        dg[0] = 0; dg[1] = (u[0] * l[0] + u[1] * l[1]) * w[0];
    }
};

// The built-in sde_lv (csrc/families.cuh SdeLotkaVolterra<false>) written in the general shape: G = diag(p4 u0, p5 u1).
// Its results agree with sde_lv's wherever the diagonal shape runs (EM + BacksolveAdjoint aside).  D = 2, P = 6, M = 2
struct SdeLotkaVolterraGeneral {
    static constexpr int D = 2, P = 6, M = 2;
    template <class T> __device__ __forceinline__ static void f(const T* u, const T* p, T* du) {
        du[0] = p[0] * u[0] - p[1] * u[0] * u[1];
        du[1] = -p[2] * u[1] + p[3] * u[0] * u[1];
    }
    template <class T> __device__ __forceinline__ static void vjp_u(const T* u, const T* p, const T* l, T* dl) {
        dl[0] = l[0] * (p[0] - p[1] * u[1]) + l[1] * p[3] * u[1];
        dl[1] = -l[0] * p[1] * u[0] + l[1] * (-p[2] + p[3] * u[0]);
    }
    template <class T> __device__ __forceinline__ static void vjp_p(const T* u, const T* p, const T* l, T* dg) {
        T xy = u[0] * u[1];
        dg[0] = u[0] * l[0]; dg[1] = -xy * l[0]; dg[2] = -u[1] * l[1]; dg[3] = xy * l[1]; dg[4] = 0; dg[5] = 0;
    }
    template <class T> __device__ __forceinline__ static void g_apply(const T* u, const T* p, const T* w, T* out) {
        out[0] = p[4] * u[0] * w[0]; out[1] = p[5] * u[1] * w[1];
    }
    template <class T> __device__ __forceinline__ static void gvjp_u_apply(const T* u, const T* p, const T* l, const T* w, T* dl) {
        dl[0] = l[0] * p[4] * w[0]; dl[1] = l[1] * p[5] * w[1];
    }
    template <class T> __device__ __forceinline__ static void gvjp_p_apply(const T* u, const T* p, const T* l, const T* w, T* dg) {
        dg[0] = 0; dg[1] = 0; dg[2] = 0; dg[3] = 0;
        dg[4] = l[0] * u[0] * w[0]; dg[5] = l[1] * u[1] * w[1];
    }
};
