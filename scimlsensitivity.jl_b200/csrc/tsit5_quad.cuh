// tsit5_quad.cuh -- QuadratureAdjoint for the fixed-step Tsit5 path: dp = sum over data intervals of
// quadgk(t -> (df/dp)(y(t))' lambda(t)) on the DENSE forward and reverse solutions (src/quadrature_adjoint.jl:486-502,
// :537-616).  One warp per member (ros23.cuh::quadgk_warp).  y(t): the forward step containing t is rebuilt from its
// checkpoint (6 RHS evaluations) and evaluated with the Tsit5 dense-output polynomials at theta = (t - t_n)/h;
// lambda(t): reverse step n stored by tsit5_reverse_kernel<SA_QUAD> as (lambda(t_{n+1}), ka'[0..6]), evaluated at
// theta_a = (t_{n+1} - t)/h.
#pragma once
#include "ode_tsit5.cuh"
#include "ros23.cuh"

namespace b200adj {

struct Tsit5QuadArgs {
    const double* ckpt; const double* adj_dense; const double* p; const double* saveat;
    double* dp_members; double* partials; double* dp; unsigned int* ticket;
    double* qseg; double* qkey; int32_t maxseg;
    int64_t N, Npad; int32_t S, K;
    double t0, t1, h, quad_abstol, quad_reltol;
    double R[7][4];          // dense-output polynomials b_j(theta) = sum_m R[j][m] theta^(m+1)
    Tsit5Tables tb;
};

template <class Fam, int D, int P>
struct Tsit5QuadCtx {
    const Tsit5QuadArgs& a; int64_t i; double p[P];
    __device__ __forceinline__ void weights(double th, double* w) const {
#pragma unroll
        for (int j = 0; j < 7; j++) w[j] = a.h * (th * (a.R[j][0] + th * (a.R[j][1] + th * (a.R[j][2] + th * a.R[j][3]))));
    }
    __device__ __forceinline__ bool valid() const { return true; }
    __device__ __forceinline__ bool empty() const { return false; }
    __device__ __forceinline__ QuadBracket root() const { return QuadBracket{0, 0, 0, 0}; }      // uniform grid: no search, no brackets
    __device__ __forceinline__ void eval(double t, const QuadBracket&, int, double* out, int* fiv, int* riv) const {
        *fiv = 0; *riv = 0;
        const int64_t cs = (int64_t)D * a.Npad;
        int n = (int)floor((t - a.t0) / a.h);
        if (n < 0) n = 0;
        if (n > a.S - 1) n = a.S - 1;
        const double tn = a.t0 + n * a.h;
        double u[D], u1[D], kf[7][D], tmp[D], y[D], lam[D], w[7];
#pragma unroll
        for (int j = 0; j < D; j++) { u[j] = a.ckpt[(int64_t)n * cs + (int64_t)j * a.Npad + i]; u1[j] = a.ckpt[(int64_t)(n + 1) * cs + (int64_t)j * a.Npad + i]; }
        Fam::f(u, p, kf[0]);
        tsit5_stage<D, 1>(a.tb, u, kf, tmp); Fam::f(tmp, p, kf[1]);
        tsit5_stage<D, 2>(a.tb, u, kf, tmp); Fam::f(tmp, p, kf[2]);
        tsit5_stage<D, 3>(a.tb, u, kf, tmp); Fam::f(tmp, p, kf[3]);
        tsit5_stage<D, 4>(a.tb, u, kf, tmp); Fam::f(tmp, p, kf[4]);
        tsit5_stage<D, 5>(a.tb, u, kf, tmp); Fam::f(tmp, p, kf[5]);
        Fam::f(u1, p, kf[6]);
        weights((t - tn) / a.h, w);
        tsit5_dense<D>(u, kf, w, y);
        const double* row = a.adj_dense + (int64_t)n * 8 * cs + i;
        double ka[7][D];
#pragma unroll
        for (int j = 0; j < D; j++) lam[j] = row[(int64_t)j * a.Npad];
#pragma unroll
        for (int s = 0; s < 7; s++)
#pragma unroll
            for (int j = 0; j < D; j++) ka[s][j] = row[((int64_t)(1 + s) * D + j) * a.Npad];
        weights(((tn + a.h) - t) / a.h, w);
        double lq[D];
        tsit5_dense<D>(lam, ka, w, lq);
        Fam::vjp_p(y, p, lq, out);
    }
};

template <class Fam, bool SHARED_P>
__global__ void __launch_bounds__(QUAD_WARPS * 32) tsit5_quadrature_kernel(const __grid_constant__ Tsit5QuadArgs a) {
    constexpr int D = Fam::D, P = Fam::P;
    quad_kernel_body<P, SHARED_P>(a, [&](int64_t i) {
        Tsit5QuadCtx<Fam, D, P> c{a, i, {}};
#pragma unroll
        for (int q = 0; q < P; q++) c.p[q] = SHARED_P ? a.p[q] : a.p[(int64_t)q * a.N + i];
        return c;
    });
}

}  // namespace b200adj
