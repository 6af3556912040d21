// ros23.cuh -- adaptive Rosenbrock23 ensemble kernels (stiff problems, BASELINE config C3): forward solve with a
// per-member dense solution, adaptive reverse adjoint solve (GaussAdjoint: 1-point Gauss per accepted step;
// QuadratureAdjoint: dense lambda + adaptive Gauss-Kronrod per data interval).  One member per thread; every member
// has its own step sequence (independent error control), so control flow diverges per lane -- the members of a warp
// are neighbouring perturbations of the same problem and stay within a few steps of each other.
//
// Reference functions replaced:
//   sense functor (lambda only)     src/quadrature_adjoint.jl:35-46, src/gauss_adjoint.jl:118-128
//   adjoint Jacobian -J(y(t))'      src/quadrature_adjoint.jl:170-192 ; d/dt of the adjoint RHS through sol(t)  :67-71
//   dense reverse solve             src/quadrature_adjoint.jl:527-530
//   AdjointSensitivityIntegrand     src/quadrature_adjoint.jl:486-502 ; interval loop :537-616 (quadgk per data interval)
//   GaussIntegrand / IntegratingSumCallback   src/gauss_adjoint.jl:745-759, :809-852
//   ReverseLossCallback             src/adjoint_common.jl:754-821
// Upstream arithmetic restated (SURVEY.md App. B): Rosenbrock23 (ode23s form, d = 1/(2+sqrt 2), e32 = 6+sqrt 2),
// its 2nd-order dense output, the I-controller (exponent 1/3, gamma 0.9, q in [0.1, 5]), QuadGK G7/K15 bisection.
#pragma once
#include <cuda_runtime.h>
#include <stdint.h>
#include "families.cuh"
#include "ode_tsit5.cuh"
#include "quadgk.cuh"

namespace b200adj {

struct RosArgs {
    // problem
    const double* u0; const double* p; const double* saveat;      // saveat[K] ascending (device)
    const double* dLdu;                                           // [K][D][N] (COST_EXPLICIT)
    double* saved;                                                // [K][D][N] or null
    int32_t* status;                                              // [N] or null: 0 ok, 1 non-finite, 2 max steps
    double* du0; double* dp_members; double* partials; double* dp; unsigned int* ticket;
    // forward dense solution (handle-owned)
    double* ft; double* fu; double* fk; int32_t* fn;              // [MAXS+1][N], [MAXS+1][D][N], [MAXS][2][D][N], [N]
    // reverse dense solution (QuadratureAdjoint), MEMBER-MAJOR: only the warp-per-member quadrature kernel reads it.
    // rrec[N][MAXS][RWP] = (t_start, h, z[D], k1[D], k2[D]) per accepted step, rend[N][MAXS] = t_start + h (the search keys)
    double* rrec; double* rend; int32_t* rn;
    // member-major copy of the forward dense solution for the same kernel (quad_transpose_fwd_kernel):
    // ftT[N][MAXS+1] knots, frecT[N][MAXS][FWP] = (u[D], k1[D], k2[D])
    double* ftT; double* frecT;
    double* qseg; double* qkey; int32_t maxseg;                  // quadgk scratch per resident warp: segments [maxseg][SEGW], keys [maxseg] (quadgk.cuh)
    int64_t N; int32_t K; int32_t maxs;
    double t0, t1, abstol, reltol, quad_abstol, quad_reltol, cost_a[4], cost_b[4];
    uint32_t flags;                                               // KF_* bits
};

__device__ constexpr double ROS_D = 0.29289321881345247559915563789515;
__device__ constexpr double ROS_E32 = 6.0 + 1.4142135623730951;
__device__ constexpr double EPS100 = 100 * 2.220446049250313e-16;

// ---- small dense LU with partial pivoting (W = I - h d J) ----
template <int D> __device__ __forceinline__ bool lu_factor(double (*A)[D], int* piv) {
#pragma unroll
    for (int c = 0; c < D; c++) {
        int pr = c; double mx = fabs(A[c][c]);
#pragma unroll
        for (int r = c + 1; r < D; r++) if (fabs(A[r][c]) > mx) { mx = fabs(A[r][c]); pr = r; }
        piv[c] = pr;
        if (mx == 0.0) return false;
        if (pr != c) {
#pragma unroll
            for (int j = 0; j < D; j++) { double t = A[c][j]; A[c][j] = A[pr][j]; A[pr][j] = t; }
        }
#pragma unroll
        for (int r = c + 1; r < D; r++) {
            double f = A[r][c] / A[c][c]; A[r][c] = f;
#pragma unroll
            for (int j = c + 1; j < D; j++) A[r][j] -= f * A[c][j];
        }
    }
    return true;
}
template <int D> __device__ __forceinline__ void lu_solve(const double (*A)[D], const int* piv, double* b) {
#pragma unroll
    for (int c = 0; c < D; c++) {
        int pr = piv[c];
        if (pr != c) { double t = b[c]; b[c] = b[pr]; b[pr] = t; }
#pragma unroll
        for (int r = c + 1; r < D; r++) b[r] -= A[r][c] * b[c];
    }
#pragma unroll
    for (int r = D - 1; r >= 0; r--) {
        double s = b[r];
#pragma unroll
        for (int j = r + 1; j < D; j++) s -= A[r][j] * b[j];
        b[r] = s / A[r][r];
    }
}

__device__ __forceinline__ double step_factor_I(double EEst) {
    double q = pow(fmax(EEst, 1e-300), 1.0 / 3.0) / 0.9;
    return fmax(0.1, fmin(5.0, q));
}
__device__ __forceinline__ double tstop_snap(double tnext, double tstop) {
    double tol = EPS100 * fmax(fabs(tnext), fabs(tstop));
    return (fabs(tnext - tstop) <= tol) ? tstop : tnext;
}

// ---- forward dense solution of one member: sol(y, t, continuity) and its time derivative ----
template <int D>
struct FwdDense {
    const double* ft; const double* fu; const double* fk; int64_t N, i; int n;
    // The adjoint solve walks the forward solution monotonically, so the interval index is kept as a CURSOR and moved by
    // linear steps (same result as a bisection over the knots, but 1-2 loads -- the two knots the interpolation needs
    // anyway -- instead of log2(n) dependent ones).
    mutable int cur = 0;
    // The interval's record (u_n, k1, k2: 3 D doubles) and its two knots stay in REGISTERS between lookups: the 3-5 lookups of
    // one adjoint step fall into one or two forward intervals, so most of them touch no memory at all.  A second register set
    // holds the interval BELOW (the solve runs downwards): its loads are issued when the current interval is entered and are
    // first used one or more steps later, so crossing a knot does not wait for global memory either (every lane has its own
    // step sequence: without this some lane of the warp misses on nearly every lookup).
    mutable int civ = -1, aiv = -1; mutable double cta = 0.0, ctb = 0.0, cu[D], ck1[D], ck2[D], ata = 0.0, au[D], ak1[D], ak2[D];
    __device__ __forceinline__ double T(int idx) const { return ft[(int64_t)idx * N + i]; }
    __device__ __forceinline__ bool holds(int iv, double ta, double tb, double t, bool right) const {
        return right ? ((iv == 0 || ta <= t) && (iv == n - 1 || tb > t)) : ((iv == 0 || ta < t) && (iv == n - 1 || tb >= t));
    }
    __device__ __forceinline__ void eval(double t, bool right, double* y, double* yd) const {
        // the cached interval is the answer exactly when the cursor search would stop on it at once
        if (!(civ >= 0 && holds(civ, cta, ctb, t, right))) {
            if (aiv >= 0 && holds(aiv, ata, cta, t, right)) {
                civ = aiv; cur = aiv; ctb = cta; cta = ata;
#pragma unroll
                for (int j = 0; j < D; j++) { cu[j] = au[j]; ck1[j] = ak1[j]; ck2[j] = ak2[j]; }
            } else {
                int iv = cur < n - 1 ? cur : n - 1;
                if (iv < 0) iv = 0;
                if (right) {        // largest idx with T(idx) <= t, clamped to [0, n-1]   (sol(t), continuity = :right)
                    while (iv > 0 && T(iv) > t) iv--;
                    while (iv < n - 1 && T(iv + 1) <= t) iv++;
                } else {            // (smallest idx with T(idx) >= t) - 1, clamped           (continuity = :left)
                    while (iv > 0 && T(iv) >= t) iv--;
                    while (iv < n - 1 && T(iv + 1) < t) iv++;
                }
                cur = iv; civ = iv;
                cta = T(iv); ctb = T(iv + 1);
#pragma unroll
                for (int j = 0; j < D; j++) {
                    cu[j] = fu[((int64_t)iv * D + j) * N + i];
                    ck1[j] = fk[(((int64_t)iv * 2 + 0) * D + j) * N + i]; ck2[j] = fk[(((int64_t)iv * 2 + 1) * D + j) * N + i];
                }
            }
            aiv = civ - 1;
            if (aiv >= 0) {       // loads of the interval below: in flight until the solve gets there
                ata = T(aiv);
#pragma unroll
                for (int j = 0; j < D; j++) {
                    au[j] = fu[((int64_t)aiv * D + j) * N + i];
                    ak1[j] = fk[(((int64_t)aiv * 2 + 0) * D + j) * N + i]; ak2[j] = fk[(((int64_t)aiv * 2 + 1) * D + j) * N + i];
                }
            }
        }
        const double ta = cta, h = ctb - ta;
        const double th = (h == 0.0) ? 1.0 : (t - ta) / h;
        const double c1 = th * (1 - th) / (1 - 2 * ROS_D), c2 = th * (th - 2 * ROS_D) / (1 - 2 * ROS_D);
        const double d1 = (1 - 2 * th) / (1 - 2 * ROS_D), d2 = (2 * th - 2 * ROS_D) / (1 - 2 * ROS_D);
#pragma unroll
        for (int j = 0; j < D; j++) {
            y[j] = cu[j] + h * (c1 * ck1[j] + c2 * ck2[j]);
            if (yd) yd[j] = d1 * ck1[j] + d2 * ck2[j];
        }
    }
};

// ------------------------------------------------------------------------------------------------------------
template <class Fam, bool SHARED_P>
__global__ void __launch_bounds__(256) ros23_forward_kernel(RosArgs a) {
    constexpr int D = Fam::D, P = Fam::P;
    const int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= a.N) return;
    const int64_t N = a.N;
    double p[P];
#pragma unroll
    for (int q = 0; q < P; q++) p[q] = SHARED_P ? a.p[q] : a.p[(int64_t)q * N + i];
    double u[D], f0[D], k1[D], k2[D], k3[D], f1[D], un[D], fn[D], tmp[D], err[D], W[D][D];
    int piv[D];
#pragma unroll
    for (int j = 0; j < D; j++) { u[j] = a.u0[(int64_t)j * N + i]; a.fu[(int64_t)j * N + i] = u[j]; }
    a.ft[i] = a.t0;
    Fam::f(u, p, f0);
    double t = a.t0, h = 1e-6 * (a.t1 - a.t0);
    int n = 0, ksave = 0, stat = 0;
    long iters = 0;
    // save times at or before t0
    while (a.saved && ksave < a.K && a.saveat[ksave] <= a.t0) {
#pragma unroll
        for (int j = 0; j < D; j++) a.saved[((int64_t)ksave * D + j) * N + i] = u[j];
        ksave++;
    }
    while (t < a.t1) {
        if (++iters > 10000000L || n >= a.maxs) { stat = 2; break; }
        bool last = false;
        if (t + h >= a.t1 || fabs(t + h - a.t1) < 100 * 2.22e-16 * fabs(a.t1)) { h = a.t1 - t; last = true; }
        // W = I - h d J ; autonomous families: dT = 0
        Fam::jac(u, p, W);
#pragma unroll
        for (int r = 0; r < D; r++)
#pragma unroll
            for (int c = 0; c < D; c++) W[r][c] = (r == c ? 1.0 : 0.0) - h * ROS_D * W[r][c];
        if (!lu_factor<D>(W, piv)) { stat = 1; break; }
#pragma unroll
        for (int j = 0; j < D; j++) k1[j] = f0[j];
        lu_solve<D>(W, piv, k1);
#pragma unroll
        for (int j = 0; j < D; j++) tmp[j] = u[j] + 0.5 * h * k1[j];
        Fam::f(tmp, p, f1);
#pragma unroll
        for (int j = 0; j < D; j++) k2[j] = f1[j] - k1[j];
        lu_solve<D>(W, piv, k2);
#pragma unroll
        for (int j = 0; j < D; j++) { k2[j] += k1[j]; un[j] = u[j] + h * k2[j]; }
        Fam::f(un, p, fn);
#pragma unroll
        for (int j = 0; j < D; j++) k3[j] = fn[j] - ROS_E32 * (k2[j] - f1[j]) - 2 * (k1[j] - f0[j]);
        lu_solve<D>(W, piv, k3);
        double e2 = 0;
#pragma unroll
        for (int j = 0; j < D; j++) {
            err[j] = h / 6.0 * (k1[j] - 2 * k2[j] + k3[j]);
            const double sc = a.abstol + a.reltol * fmax(fabs(u[j]), fabs(un[j]));
            e2 += (err[j] / sc) * (err[j] / sc);
        }
        const double EEst = sqrt(e2 / D);
        const double q = step_factor_I(EEst);
        if (EEst <= 1.0) {
            const double tn = last ? a.t1 : t + h;
            // primal at save times inside (t, tn] from this step's dense output (sol(ts), left-continuous lookup)
            while (a.saved && ksave < a.K && a.saveat[ksave] <= tn) {
                const double hh = tn - t, th = (hh == 0.0) ? 1.0 : (a.saveat[ksave] - t) / hh;
                const double c1 = th * (1 - th) / (1 - 2 * ROS_D), c2 = th * (th - 2 * ROS_D) / (1 - 2 * ROS_D);
#pragma unroll
                for (int j = 0; j < D; j++) a.saved[((int64_t)ksave * D + j) * N + i] = u[j] + hh * (c1 * k1[j] + c2 * k2[j]);
                ksave++;
            }
#pragma unroll
            for (int j = 0; j < D; j++) {
                a.fk[(((int64_t)n * 2 + 0) * D + j) * N + i] = k1[j];
                a.fk[(((int64_t)n * 2 + 1) * D + j) * N + i] = k2[j];
                a.fu[((int64_t)(n + 1) * D + j) * N + i] = un[j];
                u[j] = un[j]; f0[j] = fn[j];
            }
            t = tn; a.ft[(int64_t)(n + 1) * N + i] = t;
            n++;
        }
        h = h / q;
    }
    a.fn[i] = n;
    bool ok = true;
#pragma unroll
    for (int j = 0; j < D; j++) ok = ok && isfinite(u[j]);
    if (!ok && stat == 0) stat = 1;
    if (a.status) a.status[i] = stat;
}

// adjoint RHS  dlam = -J(y(t))' lam  (right-continuous forward lookup) and, on request, its Jacobian / time derivative
template <class Fam, int D>
__device__ __forceinline__ void adj_rhs(const FwdDense<D>& sol, const double* p, double t, const double* lam, double* out) {
    double y[D];
    sol.eval(t, true, y, nullptr);
    Fam::vjp_u(y, p, lam, out);
#pragma unroll
    for (int j = 0; j < D; j++) out[j] = -out[j];
}

template <class Fam, int SA, bool SHARED_P, int COST>
__global__ void __launch_bounds__(256) ros23_reverse_kernel(RosArgs a) {
    constexpr int D = Fam::D, P = Fam::P;
    const int64_t gi = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
    const bool active = gi < a.N;
    const int64_t i = active ? gi : a.N - 1;
    const int64_t N = a.N;
    double p[P], acc[P];
#pragma unroll
    for (int q = 0; q < P; q++) { p[q] = SHARED_P ? a.p[q] : a.p[(int64_t)q * N + i]; acc[q] = 0.0; }
    FwdDense<D> sol{a.ft, a.fu, a.fk, N, i, a.fn[i]};
    sol.cur = sol.n - 1;                  // the reverse solve starts at T
    double z[D], zn[D], f0[D], k1[D], k2[D], k3[D], f1[D], fnr[D], tmp[D], W[D][D], dT[D];
    int piv[D];
#pragma unroll
    for (int j = 0; j < D; j++) z[j] = 0.0;
    const double T = a.t1, t0 = a.t0;
    double t = T;
    int cur = a.K - 1, nrev = 0;
    bool fsal_ok = false, overflow = false;
    auto jump_if_at = [&](double tt) {
        while (cur >= 0 && fabs(a.saveat[cur] - tt) <= EPS100 * fmax(fabs(tt), 1.0)) {
            if (!((a.flags & KF_NO_START) && cur == 0)) {
                double y[D];
                if (COST == COST_EXPLICIT) {
#pragma unroll
                    for (int j = 0; j < D; j++) z[j] += a.dLdu[((int64_t)cur * D + j) * N + i];
                } else {
                    sol.eval(a.saveat[cur], true, y, nullptr);
#pragma unroll
                    for (int j = 0; j < D; j++) z[j] += a.cost_a[j] * y[j] + a.cost_b[j];
                }
            }
            cur--; fsal_ok = false;
        }
    };
    jump_if_at(t);
    double h = -1e-4 * (T - t0);
    long iters = 0;
    while (t > t0 && sol.n > 0) {
        if (++iters > 50000000L || (SA == SA_QUAD && nrev >= a.maxs)) { overflow = true; break; }
        double tstop = t0;
        if (cur >= 0 && a.saveat[cur] < t && a.saveat[cur] > tstop) tstop = a.saveat[cur];
        double tn = tstop_snap(t + h, tstop);
        if (tn < tstop) tn = tstop;
        const double hs = tn - t;
        if (!fsal_ok) adj_rhs<Fam, D>(sol, p, t, z, f0);
        // Jacobian of the adjoint RHS wrt lambda (-J') and its time derivative -(dJ/dt)' lambda, ydot from the interpolant
        {
            double y[D], yd[D], J[D][D], dJ[D][D];
            sol.eval(t, true, y, yd);
            Fam::jac(y, p, J); Fam::djac(p, yd, dJ);
#pragma unroll
            for (int r = 0; r < D; r++) {
                double s = 0;
#pragma unroll
                for (int c = 0; c < D; c++) { W[r][c] = (r == c ? 1.0 : 0.0) - hs * ROS_D * (-J[c][r]); s -= dJ[c][r] * z[c]; }
                dT[r] = s;
            }
        }
        if (!lu_factor<D>(W, piv)) break;
#pragma unroll
        for (int j = 0; j < D; j++) k1[j] = f0[j] + hs * ROS_D * dT[j];
        lu_solve<D>(W, piv, k1);
#pragma unroll
        for (int j = 0; j < D; j++) tmp[j] = z[j] + 0.5 * hs * k1[j];
        adj_rhs<Fam, D>(sol, p, t + 0.5 * hs, tmp, f1);
#pragma unroll
        for (int j = 0; j < D; j++) k2[j] = f1[j] - k1[j];
        lu_solve<D>(W, piv, k2);
#pragma unroll
        for (int j = 0; j < D; j++) { k2[j] += k1[j]; zn[j] = z[j] + hs * k2[j]; }
        adj_rhs<Fam, D>(sol, p, t + hs, zn, fnr);
#pragma unroll
        for (int j = 0; j < D; j++) k3[j] = fnr[j] - ROS_E32 * (k2[j] - f1[j]) - 2 * (k1[j] - f0[j]) + hs * ROS_D * dT[j];
        lu_solve<D>(W, piv, k3);
        double e2 = 0;
#pragma unroll
        for (int j = 0; j < D; j++) {
            const double e = hs / 6.0 * (k1[j] - 2 * k2[j] + k3[j]);
            const double sc = a.abstol + a.reltol * fmax(fabs(z[j]), fabs(zn[j]));
            e2 += (e / sc) * (e / sc);
        }
        const double EEst = sqrt(e2 / D);
        const double q = step_factor_I(EEst);
        if (EEst > 1.0) { h = hs / q; fsal_ok = true; continue; }
        h = hs / q;
        if (SA == SA_GAUSS) {
            // IntegratingSumCallback, n = (alg_order+1) div 2 = 1 node: midpoint, weight 2, scale (tn - t)/2, integrand -F'lam
            const double tj = 0.5 * (tn + t), th = (tj - t) / hs;
            const double c1 = th * (1 - th) / (1 - 2 * ROS_D), c2 = th * (th - 2 * ROS_D) / (1 - 2 * ROS_D);
            double lq[D], y[D], dg[P];
#pragma unroll
            for (int j = 0; j < D; j++) lq[j] = z[j] + hs * (c1 * k1[j] + c2 * k2[j]);
            sol.eval(tj, false, y, nullptr);
            Fam::vjp_p(y, p, lq, dg);
#pragma unroll
            for (int q2 = 0; q2 < P; q2++) acc[q2] += (0.5 * (tn - t)) * 2.0 * (-dg[q2]);
        } else if (SA == SA_GK) {
            auto node = [&](double tj, double* out) {
                const double th = (tj - t) / hs;
                const double c1 = th * (1 - th) / (1 - 2 * ROS_D), c2 = th * (th - 2 * ROS_D) / (1 - 2 * ROS_D);
                double lq[D], y[D];
#pragma unroll
                for (int j = 0; j < D; j++) lq[j] = z[j] + hs * (c1 * k1[j] + c2 * k2[j]);
                sol.eval(tj, false, y, nullptr);
                Fam::vjp_p(y, p, lq, out);
#pragma unroll
                for (int q2 = 0; q2 < P; q2++) out[q2] = -out[q2];
            };
            integrate_gk_step<P, 1>(node, t, tn, acc);
        } else if (active) {
            double* rec = a.rrec + ((int64_t)i * a.maxs + nrev) * quad_pad(3 + 3 * D);
            rec[0] = t; rec[1] = hs; rec[2 + 3 * D] = 1.0 / hs;
            a.rend[(int64_t)i * a.maxs + nrev] = t + hs;
#pragma unroll
            for (int j = 0; j < D; j++) { rec[2 + j] = z[j]; rec[2 + D + j] = k1[j]; rec[2 + 2 * D + j] = k2[j]; }
        }
        nrev++;
#pragma unroll
        for (int j = 0; j < D; j++) { z[j] = zn[j]; f0[j] = fnr[j]; }
        fsal_ok = true;
        t = tn;
        jump_if_at(t);
    }
    if (active) {
        // a member whose dense reverse solution did not fit (max steps) fails loudly: NaN gradient, never a silent partial
#pragma unroll
        for (int j = 0; j < D; j++) a.du0[(int64_t)j * N + i] = overflow ? __longlong_as_double(0x7ff8000000000000LL) : z[j];
        if (SA == SA_QUAD) a.rn[i] = overflow ? -1 : nrev;
    }
    if (SA == SA_GAUSS || SA == SA_GK) {
        if (SHARED_P) {
            if (!active) {
#pragma unroll
                for (int q = 0; q < P; q++) acc[q] = 0.0;
            }
            reduce_dp<P>(acc, a.partials, a.dp, a.ticket);
        } else if (active) {
#pragma unroll
            for (int q = 0; q < P; q++) a.dp_members[(int64_t)q * N + i] = acc[q];
        }
    }
}

// ------------------------------------------------------------------------------------------------------------
// Rosenbrock23 on the AUGMENTED adjoint states: InterpolatingAdjoint z = [lam; mu] and BacksolveAdjoint z = [lam; mu; y]
// (src/interpolating_adjoint.jl:150-174, src/backsolve_adjoint.jl:32-61; the reference runs every sensealg with stiff solvers,
// test/Core2/stiff_adjoints.jl:204-252).  W = I - h d (d rhs / dz) is block triangular, so the linear solves are the 3 x 3 LU
// of the lambda block (and of the y block for Backsolve) plus substitutions:
//   Interpolating   W = [[I + hd J', 0], [hd F', I]]                         dT = [-(dJ/dt)'lam, -(dF/dt)'lam]   (ydot from sol)
//   Backsolve       W = [[I + hd J', 0, hd H], [hd F', I, hd G], [0, 0, I - hd J]]   autonomous: dT = 0
//                   H v = d(J'lam)/dy [v], G v = d(F'lam)/dy [v]  (families.cuh::djac, dvjp_p)
// Error norm over all components of z (the reference's augmented state).  Checkpoints / jumps as in t5a_reverse_kernel.
// ------------------------------------------------------------------------------------------------------------
template <class Fam, int SA, bool SHARED_P, int COST>
__global__ void __launch_bounds__(256) ros23_aug_reverse_kernel(RosArgs a) {
    static_assert(SA == SA_INTERP || SA == SA_BACKSOLVE, "augmented states only");
    constexpr int D = Fam::D, P = Fam::P, L = (SA == SA_INTERP) ? D + P : 2 * D + P, YO = D + P;
    const int64_t gi = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
    const bool active = gi < a.N;
    const int64_t i = active ? gi : a.N - 1;
    const int64_t N = a.N;
    double p[P];
#pragma unroll
    for (int q = 0; q < P; q++) p[q] = SHARED_P ? a.p[q] : a.p[(int64_t)q * N + i];
    FwdDense<D> sol{a.ft, a.fu, a.fk, N, i, a.fn[i]};
    sol.cur = sol.n - 1;
    double z[L], zn[L], f0[L], k1[L], k2[L], k3[L], f1[L], fnr[L], tmp[L], dT[L];
    double Wl[D][D], Wy[D][D], yj[D], lamj[D];            // Jacobian point of the current step (y, lam at t)
    int pivl[D], pivy[D];
#pragma unroll
    for (int c = 0; c < L; c++) { z[c] = 0.0; dT[c] = 0.0; }
    auto rhs = [&](double tt, const double* x, double* dx) {
        double y[D], dg[P];
        if (SA == SA_BACKSOLVE) {
#pragma unroll
            for (int j = 0; j < D; j++) y[j] = x[YO + j];
        } else sol.eval(tt, true, y, nullptr);
        Fam::vjp_u(y, p, x, dx);
        Fam::vjp_p(y, p, x, dg);
#pragma unroll
        for (int j = 0; j < D; j++) dx[j] = -dx[j];
#pragma unroll
        for (int q = 0; q < P; q++) dx[D + q] = -dg[q];
        if (SA == SA_BACKSOLVE) Fam::f(y, p, dx + YO);
    };
    double hd = 0.0;                                     // hs * d of the current step
    auto solveW = [&](double* b) {
        double dg[P];
        if (SA == SA_BACKSOLVE) {
            lu_solve<D>(Wy, pivy, b + YO);
            double dJ[D][D];
            Fam::djac(p, b + YO, dJ);
#pragma unroll
            for (int r = 0; r < D; r++) {
                double s = 0;
#pragma unroll
                for (int c = 0; c < D; c++) s += dJ[c][r] * lamj[c];
                b[r] -= hd * s;
            }
        }
        lu_solve<D>(Wl, pivl, b);
        Fam::vjp_p(yj, p, b, dg);
#pragma unroll
        for (int q = 0; q < P; q++) b[D + q] -= hd * dg[q];
        if (SA == SA_BACKSOLVE) {
            Fam::dvjp_p(yj, p, b + YO, lamj, dg);
#pragma unroll
            for (int q = 0; q < P; q++) b[D + q] -= hd * dg[q];
        }
    };
    const double T = a.t1, t0 = a.t0;
    double t = T;
    int cur = a.K - 1, ck = sol.n;
    bool fsal_ok = false, failed = false;
    const bool ckpt_on = !(a.flags & KF_NO_CHECKPOINTING), every = (a.flags & KF_CKPT_EVERY_STEP);
    if (SA == SA_BACKSOLVE) {
#pragma unroll
        for (int j = 0; j < D; j++) z[YO + j] = a.fu[((int64_t)sol.n * D + j) * N + i];     // y(T) = sol.u[end]
    }
    auto ckpt_if_at = [&](double tt) {                   // Backsolve checkpoint callback: y <- sol(t) (runs before the loss jump)
        if (SA != SA_BACKSOLVE || !ckpt_on) return;
        const double tol = EPS100 * fmax(fabs(tt), 1.0);
        if (every) {
            while (ck >= 0 && sol.T(ck) > tt + tol) ck--;
            if (ck >= 0 && fabs(sol.T(ck) - tt) <= tol) {
#pragma unroll
                for (int j = 0; j < D; j++) z[YO + j] = a.fu[((int64_t)ck * D + j) * N + i];
                fsal_ok = false;
            }
        } else if (cur >= 0 && fabs(a.saveat[cur] - tt) <= tol) {
            double y[D];
            sol.eval(a.saveat[cur], true, y, nullptr);
#pragma unroll
            for (int j = 0; j < D; j++) z[YO + j] = y[j];
            fsal_ok = false;
        }
    };
    auto jump_if_at = [&](double tt) {
        while (cur >= 0 && fabs(a.saveat[cur] - tt) <= EPS100 * fmax(fabs(tt), 1.0)) {
            if (!((a.flags & KF_NO_START) && cur == 0 && SA != SA_BACKSOLVE)) {
                if (COST == COST_EXPLICIT) {
#pragma unroll
                    for (int j = 0; j < D; j++) z[j] += a.dLdu[((int64_t)cur * D + j) * N + i];
                } else {
                    double y[D];
                    if (SA == SA_BACKSOLVE) {
#pragma unroll
                        for (int j = 0; j < D; j++) y[j] = z[YO + j];
                    } else sol.eval(a.saveat[cur], true, y, nullptr);
#pragma unroll
                    for (int j = 0; j < D; j++) z[j] += a.cost_a[j] * y[j] + a.cost_b[j];
                }
            }
            cur--; fsal_ok = false;
        }
    };
    ckpt_if_at(t);
    jump_if_at(t);
    double h = -1e-4 * (T - t0);
    long iters = 0;
    while (t > t0 && sol.n > 0) {
        if (++iters > 50000000L) { failed = true; break; }
        double tstop = t0;
        if (cur >= 0 && a.saveat[cur] < t && a.saveat[cur] > tstop) tstop = a.saveat[cur];
        if (SA == SA_BACKSOLVE && ckpt_on && every) {            // every forward knot is a tstop of the reverse solve
            int c2 = ck;
            while (c2 >= 0 && sol.T(c2) >= t - EPS100 * fmax(fabs(t), 1.0)) c2--;
            if (c2 >= 0 && sol.T(c2) > tstop) tstop = sol.T(c2);
        }
        double tn = tstop_snap(t + h, tstop);
        if (tn < tstop) tn = tstop;
        const double hs = tn - t;
        hd = hs * ROS_D;
        if (!fsal_ok) rhs(t, z, f0);
        {   // Jacobian blocks and the time derivative at (t, z)
            double yd[D], J[D][D], dJ[D][D], dg[P];
            if (SA == SA_BACKSOLVE) {
#pragma unroll
                for (int j = 0; j < D; j++) { yj[j] = z[YO + j]; yd[j] = 0.0; }
            } else sol.eval(t, true, yj, yd);
#pragma unroll
            for (int j = 0; j < D; j++) lamj[j] = z[j];
            Fam::jac(yj, p, J);
#pragma unroll
            for (int r = 0; r < D; r++)
#pragma unroll
                for (int c = 0; c < D; c++) { Wl[r][c] = (r == c ? 1.0 : 0.0) + hd * J[c][r]; Wy[r][c] = (r == c ? 1.0 : 0.0) - hd * J[r][c]; }
            if (SA == SA_INTERP) {
                Fam::djac(p, yd, dJ);
                Fam::dvjp_p(yj, p, yd, lamj, dg);
#pragma unroll
                for (int r = 0; r < D; r++) {
                    double s = 0;
#pragma unroll
                    for (int c = 0; c < D; c++) s -= dJ[c][r] * lamj[c];
                    dT[r] = s;
                }
#pragma unroll
                for (int q = 0; q < P; q++) dT[D + q] = -dg[q];
            }
        }
        if (!lu_factor<D>(Wl, pivl) || (SA == SA_BACKSOLVE && !lu_factor<D>(Wy, pivy))) { failed = true; break; }
#pragma unroll
        for (int c = 0; c < L; c++) k1[c] = f0[c] + hd * dT[c];
        solveW(k1);
#pragma unroll
        for (int c = 0; c < L; c++) tmp[c] = z[c] + 0.5 * hs * k1[c];
        rhs(t + 0.5 * hs, tmp, f1);
#pragma unroll
        for (int c = 0; c < L; c++) k2[c] = f1[c] - k1[c];
        solveW(k2);
#pragma unroll
        for (int c = 0; c < L; c++) { k2[c] += k1[c]; zn[c] = z[c] + hs * k2[c]; }
        rhs(t + hs, zn, fnr);
#pragma unroll
        for (int c = 0; c < L; c++) k3[c] = fnr[c] - ROS_E32 * (k2[c] - f1[c]) - 2 * (k1[c] - f0[c]) + hd * dT[c];
        solveW(k3);
        double e2 = 0;
#pragma unroll
        for (int c = 0; c < L; c++) {
            const double e = hs / 6.0 * (k1[c] - 2 * k2[c] + k3[c]);
            const double sc = a.abstol + a.reltol * fmax(fabs(z[c]), fabs(zn[c]));
            e2 += (e / sc) * (e / sc);
        }
        const double EEst = sqrt(e2 / L);
        if (!isfinite(EEst)) { failed = true; break; }           // e.g. Backsolve blowing up backwards on a stiff problem
        const double q = step_factor_I(EEst);
        if (EEst > 1.0) { h = hs / q; fsal_ok = true; continue; }
        h = hs / q;
#pragma unroll
        for (int c = 0; c < L; c++) { z[c] = zn[c]; f0[c] = fnr[c]; }
        fsal_ok = true;
        t = tn;
        ckpt_if_at(t);
        jump_if_at(t);
    }
    const double qnan = __longlong_as_double(0x7ff8000000000000LL);
    if (active) {
#pragma unroll
        for (int j = 0; j < D; j++) a.du0[(int64_t)j * N + i] = failed ? qnan : z[j];
    }
    double out[P];
#pragma unroll
    for (int q = 0; q < P; q++) out[q] = failed ? qnan : z[D + q];
    if (SHARED_P) {
        if (!active) {
#pragma unroll
            for (int q = 0; q < P; q++) out[q] = 0.0;
        }
        reduce_dp<P>(out, a.partials, a.dp, a.ticket);
    } else if (active) {
#pragma unroll
        for (int q = 0; q < P; q++) a.dp_members[(int64_t)q * N + i] = out[q];
    }
}

// QuadratureAdjoint integrand on the two dense solutions (AdjointSensitivityIntegrand, src/quadrature_adjoint.jl:486-502):
// out = (df/dp)(y(t))' lam(t), y left-continuous from the forward dense solution, lam from the dense reverse solution.
// The lookups are warp-cooperative inside the segment's index brackets (quadgk.cuh).
template <class Fam, int D, int P>
struct RosQuadCtx {
    static constexpr int FWP = quad_pad(3 * D + 3), RWP = quad_pad(3 + 3 * D);
    const double* ftT; const double* frecT; const double* rrec; const double* rend;      // this member's rows
    int nf, nrev; double p[P];
    __device__ __forceinline__ bool valid() const { return nrev >= 0; }
    __device__ __forceinline__ bool empty() const { return nrev == 0; }
    __device__ __forceinline__ QuadBracket root() const { return QuadBracket{0, nf - 1, 0, nrev - 1}; }
    __device__ __forceinline__ void eval(double t, const QuadBracket& br, int lane, double* out, int* fiv, int* riv) const {
        double y[D], lam[D];
        constexpr double IC = 1.0 / (1 - 2 * ROS_D);
        // forward: iv = #{interior knots < t} (sol(y, t, continuity = :left))
        const int iv = br.flo + coop_count<true>([&](int j) { return __ldg(ftT + j); }, br.flo + 1, br.fhi - br.flo, t, lane);
        // reverse: the step whose end is the first <= t; ends descend with the step index
        const int lo = br.rlo + coop_count<false>([&](int j) { return __ldg(rend + j); }, br.rlo, br.rhi - br.rlo, t, lane);
        *fiv = iv; *riv = lo;
        {
            const double* r = frecT + iv * FWP;                  // (u[D], k1[D], k2[D], t_a, h, 1/h)
            const double ta = __ldg(r + 3 * D), h = __ldg(r + 3 * D + 1), ih = __ldg(r + 3 * D + 2);
            const double th = (h == 0.0) ? 1.0 : (t - ta) * ih;
            const double c1 = th * (1 - th) * IC, c2 = th * (th - 2 * ROS_D) * IC;
#pragma unroll
            for (int j = 0; j < D; j++) y[j] = __ldg(r + j) + h * (c1 * __ldg(r + D + j) + c2 * __ldg(r + 2 * D + j));
        }
        {
            const double* r = rrec + lo * RWP;                   // (t_start, h, z[D], k1[D], k2[D], 1/h)
            const double ts = __ldg(r), h = __ldg(r + 1), th = (t - ts) * __ldg(r + 2 + 3 * D);
            const double c1 = th * (1 - th) * IC, c2 = th * (th - 2 * ROS_D) * IC;
#pragma unroll
            for (int j = 0; j < D; j++) lam[j] = __ldg(r + 2 + j) + h * (c1 * __ldg(r + 2 + D + j) + c2 * __ldg(r + 2 + 2 * D + j));
        }
        Fam::vjp_p(y, p, lam, out);
    }
};

// persistent grid of 4-warp blocks, one warp per member at a time (quadgk.cuh::quad_member_loop)
template <class Fam, bool SHARED_P>
__global__ void __launch_bounds__(QUAD_WARPS * 32) ros23_quadrature_kernel(RosArgs a) {
    constexpr int D = Fam::D, P = Fam::P;
    extern __shared__ double s_quad_l1[];
    const int lane = threadIdx.x & 31;
    const int64_t N = a.N;
    double acc[P];
#pragma unroll
    for (int q = 0; q < P; q++) acc[q] = 0.0;
    auto make = [&](int64_t i) {
        RosQuadCtx<Fam, D, P> c{a.ftT + (int64_t)i * (a.maxs + 1), a.frecT + (int64_t)i * a.maxs * quad_pad(3 * D + 3),
                                a.rrec + (int64_t)i * a.maxs * quad_pad(3 + 3 * D), a.rend + (int64_t)i * a.maxs, a.fn[i], a.rn[i], {}};
#pragma unroll
        for (int q = 0; q < P; q++) c.p[q] = SHARED_P ? a.p[q] : a.p[(int64_t)q * N + i];
        return c;
    };
    auto sink = [&](int64_t i, const double* res) {
        if (SHARED_P) {
#pragma unroll
            for (int q = 0; q < P; q++) acc[q] += res[q];
        } else if (lane == 0) {
#pragma unroll
            for (int q = 0; q < P; q++) a.dp_members[(int64_t)q * N + i] = res[q];
        }
    };
    quad_member_loop<P>(N, a.K, a.saveat, a.t0, a.t1, a.quad_abstol, a.quad_reltol, a.qseg, a.qkey, a.maxseg, s_quad_l1, make, sink);
    if (SHARED_P) {
        if (lane != 0) {
#pragma unroll
            for (int q = 0; q < P; q++) acc[q] = 0.0;
        }
        reduce_dp<P>(acc, a.partials, a.dp, a.ticket);
    }
}

}  // namespace b200adj
