// sde_families.cuh -- USER diagonal-noise SDE families for libb200adj.so (not part of the library), in the shape of
// SdeLotkaVolterra in csrc/families.cuh: du = f(u, p) dt + g(u, p) .* dW, one Wiener process per state, g_i a function of u_i
// and p only.  ITO = true gives the Ito-transformed drift F_i = f_i - g_i dg_i/du_i (src/sde_tools.jl:29-66) and its VJPs,
// which BacksolveAdjoint runs with the Ito solver EM; EulerHeun, InterpolatingAdjoint and the forward pass run ITO = false.
// Build + register:  python -m scimlsensitivity_jl_b200.family_plugin examples/sde_families.cuh SdeFoodChain3 sde_chain3 --sde
#pragma once

// Three-species Lotka-Volterra food chain with saturating noise            d = 3, P = 6, M = 3 (one half-used Philox pair)
//   f = (u0 (p0 - u1),  u1 (u0 - p1 - u2),  u2 (u1 - p2)),   g_i = p_{3+i} r(u_i),  r(u) = u / (1 + u^2)
// r'' != 0, so the Ito correction g_i g_i' = p_{3+i}^2 c(u_i), c = r r' = u (1 - u^2) / (1 + u^2)^3, is not linear in u.
template <bool ITO>
struct SdeFoodChain3 {
    static constexpr int D = 3, P = 6, M = 3;
    template <class T> __device__ __forceinline__ static T r(T u) { return u / (1 + u * u); }
    template <class T> __device__ __forceinline__ static T dr(T u) { const T q = 1 + u * u; return (1 - u * u) / (q * q); }
    template <class T> __device__ __forceinline__ static T c(T u) { const T q = 1 + u * u; return u * (1 - u * u) / (q * q * q); }
    template <class T> __device__ __forceinline__ static T dc(T u) {
        const T q = 1 + u * u, u2 = u * u;
        return (1 - 8 * u2 + 3 * u2 * u2) / (q * q * q * q);
    }
    template <class T> __device__ __forceinline__ static void f(const T* u, const T* p, T* du) {
        du[0] = u[0] * (p[0] - u[1]);
        du[1] = u[1] * (u[0] - p[1] - u[2]);
        du[2] = u[2] * (u[1] - p[2]);
        if (ITO) {
#pragma unroll
            for (int i = 0; i < 3; i++) du[i] -= p[3 + i] * p[3 + i] * c(u[i]);
        }
    }
    template <class T> __device__ __forceinline__ static void g(const T* u, const T* p, T* g) {
#pragma unroll
        for (int i = 0; i < 3; i++) g[i] = p[3 + i] * r(u[i]);
    }
    // dl = (df/du)' l
    template <class T> __device__ __forceinline__ static void vjp_u(const T* u, const T* p, const T* l, T* dl) {
        dl[0] = l[0] * (p[0] - u[1]) + l[1] * u[1];
        dl[1] = -l[0] * u[0] + l[1] * (u[0] - p[1] - u[2]) + l[2] * u[2];
        dl[2] = -l[1] * u[1] + l[2] * (u[1] - p[2]);
        if (ITO) {
#pragma unroll
            for (int i = 0; i < 3; i++) dl[i] -= p[3 + i] * p[3 + i] * dc(u[i]) * l[i];
        }
    }
    // dg = (df/dp)' l
    template <class T> __device__ __forceinline__ static void vjp_p(const T* u, const T* p, const T* l, T* dg) {
        dg[0] = u[0] * l[0]; dg[1] = -u[1] * l[1]; dg[2] = -u[2] * l[2];
#pragma unroll
        for (int i = 0; i < 3; i++) dg[3 + i] = ITO ? -2 * p[3 + i] * c(u[i]) * l[i] : T(0);
    }
    // dl_i = l_i dg_i/du_i
    template <class T> __device__ __forceinline__ static void gvjp_u(const T* u, const T* p, const T* l, T* dl) {
#pragma unroll
        for (int i = 0; i < 3; i++) dl[i] = l[i] * p[3 + i] * dr(u[i]);
    }
    // dgw = sum_i l_i (dg_i/dp) w_i: column i has one non-zero, row 3 + i, value r(u_i)
    template <class T> __device__ __forceinline__ static void gvjp_p_apply(const T* u, const T* p, const T* l, const T* w, T* dgw) {
        dgw[0] = 0; dgw[1] = 0; dgw[2] = 0;
#pragma unroll
        for (int i = 0; i < 3; i++) dgw[3 + i] = l[i] * r(u[i]) * w[i];
    }
};

// Two coupled oscillators, the second with a cubic spring, and noise growing with the state   d = 4, P = 8, M = 4
//   f = (u1,  -p0 u0 - p1 u1 + p2 (u2 - u0),  u3,  -p3 u2^3 + p2 (u0 - u2)),   g_i = p_{4+i} (1 + u_i^2)
// the registry's limits (D = 4, P = 8); Ito correction g_i g_i' = p_{4+i}^2 c(u_i), c = 2 u (1 + u^2)
template <bool ITO>
struct SdeOscillator4 {
    static constexpr int D = 4, P = 8, M = 4;
    template <class T> __device__ __forceinline__ static T c(T u) { return 2 * u * (1 + u * u); }
    template <class T> __device__ __forceinline__ static T dc(T u) { return 2 + 6 * u * u; }
    template <class T> __device__ __forceinline__ static void f(const T* u, const T* p, T* du) {
        du[0] = u[1];
        du[1] = -p[0] * u[0] - p[1] * u[1] + p[2] * (u[2] - u[0]);
        du[2] = u[3];
        du[3] = -p[3] * u[2] * u[2] * u[2] + p[2] * (u[0] - u[2]);
        if (ITO) {
#pragma unroll
            for (int i = 0; i < 4; i++) du[i] -= p[4 + i] * p[4 + i] * c(u[i]);
        }
    }
    template <class T> __device__ __forceinline__ static void g(const T* u, const T* p, T* g) {
#pragma unroll
        for (int i = 0; i < 4; i++) g[i] = p[4 + i] * (1 + u[i] * u[i]);
    }
    template <class T> __device__ __forceinline__ static void vjp_u(const T* u, const T* p, const T* l, T* dl) {
        dl[0] = -(p[0] + p[2]) * l[1] + p[2] * l[3];
        dl[1] = l[0] - p[1] * l[1];
        dl[2] = p[2] * l[1] - (3 * p[3] * u[2] * u[2] + p[2]) * l[3];
        dl[3] = l[2];
        if (ITO) {
#pragma unroll
            for (int i = 0; i < 4; i++) dl[i] -= p[4 + i] * p[4 + i] * dc(u[i]) * l[i];
        }
    }
    template <class T> __device__ __forceinline__ static void vjp_p(const T* u, const T* p, const T* l, T* dg) {
        dg[0] = -u[0] * l[1];
        dg[1] = -u[1] * l[1];
        dg[2] = (u[2] - u[0]) * (l[1] - l[3]);
        dg[3] = -u[2] * u[2] * u[2] * l[3];
#pragma unroll
        for (int i = 0; i < 4; i++) dg[4 + i] = ITO ? -2 * p[4 + i] * c(u[i]) * l[i] : T(0);
    }
    template <class T> __device__ __forceinline__ static void gvjp_u(const T* u, const T* p, const T* l, T* dl) {
#pragma unroll
        for (int i = 0; i < 4; i++) dl[i] = l[i] * p[4 + i] * 2 * u[i];
    }
    template <class T> __device__ __forceinline__ static void gvjp_p_apply(const T* u, const T* p, const T* l, const T* w, T* dgw) {
        dgw[0] = 0; dgw[1] = 0; dgw[2] = 0; dgw[3] = 0;
#pragma unroll
        for (int i = 0; i < 4; i++) dgw[4 + i] = l[i] * (1 + u[i] * u[i]) * w[i];
    }
};
