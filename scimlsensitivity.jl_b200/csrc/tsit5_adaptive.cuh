// tsit5_adaptive.cuh -- error-controlled Tsit5 (the reference's default non-stiff solver, BASELINE config C1) on the
// per-member adaptive framework of ros23.cuh: forward solve with a per-member dense solution (t_n, u_n, k1..k7), adaptive
// reverse adjoint solve for InterpolatingAdjoint (z = [lambda; mu]), GaussAdjoint (3-point Gauss-Legendre per accepted
// step) and QuadratureAdjoint (dense lambda, then ros23.cuh::quadgk_warp).  One member per thread.
//
// Reference functions replaced: src/interpolating_adjoint.jl:150-174, src/gauss_adjoint.jl:118-128, :745-759,
// src/quadrature_adjoint.jl:35-46, :486-502, :537-616, split_states sol(y,t,continuity=:right), ReverseLossCallback
// src/adjoint_common.jl:754-821.  Upstream arithmetic restated (SURVEY.md App. B): Tsit5 tableau, embedded error
// weights, 4th-order dense output, PI controller (beta1 = 7/50, beta2 = 2/25, gamma = 0.9, q in [1/10, 5], qoldinit 1e-4).
#pragma once
#include <cuda_runtime.h>
#include <stdint.h>
#include "families.cuh"
#include "ode_tsit5.cuh"
#include "ros23.cuh"

namespace b200adj {

struct T5aArgs {
    const double* u0; const double* p; const double* saveat; const double* dLdu;
    double* saved; int32_t* status;
    double* du0; double* dp_members; double* partials; double* dp; unsigned int* ticket;
    double* ft; double* fu; double* fk; int32_t* fn;              // fn[N]: accepted forward steps per member (ft / fu / fk: unused by these kernels)
    double* rrec; double* rend; int32_t* rn;                      // reverse dense (Quadrature), member-major: [N][MAXS][RWP] = (t, h, z[D], k[7][D]), [N][MAXS] = t + h
    // THE forward dense solution, member-major: every member has its own step sequence, so its records are contiguous and move
    // as ONE bulk copy each (TMA): knots ftT[N][MAXS+1]; records frecT[N][MAXS+1][8 D + 4] = (u_n[D], c0..c3[D] = the interpolant in powers of theta, 3 D unused, t_n, h, 1/h,
    // t_{n+1}); record fn[i] (the last) holds the final state and time only
    double* ftT; double* frecT;
    double* qseg; double* qkey; int32_t maxseg;
    int64_t N; int32_t K; int32_t maxs;
    double t0, t1, dt0, abstol, reltol, quad_abstol, quad_reltol, cost_a[4], cost_b[4];
    uint32_t flags;
    // preset-time events u <- scale .* u + shift (the hybrid-system adjoint of src/callback_tracking.jl:232-480 for the
    // affine affect family, save_positions = (false, false)): same events for every member, times ascending in (t0, t1)
    int32_t nev; const double* ev_t; const double* ev_s; const double* ev_c;      // [E], [E][D], [E][D]
    double cont_a[4], cont_b[4];  // KF_CONT_COST: continuous cost g(u) = cont_a/2 |u|^2 + cont_b sum(u), dlam -= dgdu_continuous(y) (accumulate_cost!)
    const double* ev_ps; const double* ev_pc;     // [E][P] or null: parameter-changing affect p <- ps .* p + pc (reset_p of the reference)
    // [E] or null: affect that adds a parameter to a state, u[ev_ac[e]] += ev_af[e] * p[ev_ak[e]] with the parameters in force before
    // the event ("Dosing example", test/Callbacks1/discrete_callbacks.jl:401-427: integrator.u[1] += integrator.p[2]); ev_ac[e] < 0: none
    const int32_t* ev_ac; const int32_t* ev_ak; const double* ev_af;
    // state-dependent event (ContinuousCallback, src/callback_tracking.jl:232-480; docs/src/examples/hybrid_jump/bouncing_ball.md):
    // condition u[cc_idx] - cc_level crossing zero in direction cc_dir (-1 down, +1 up, 0 both); affect u <- cc_scale .* u +
    // cc_shift, then u[cc_pcomp] <- cc_psign * p[cc_pparam] * u[cc_pcomp] (cc_pcomp < 0: none).  The forward kernel (CC = true)
    // FINDS each member's event times: cc_t[cc_maxev][N], cc_n[N]; the reverse kernel reads them as member-local tstops.
    int32_t cc_on, cc_idx, cc_dir, cc_pcomp, cc_pparam, cc_maxev;
    double cc_level, cc_psign, cc_scale[4], cc_shift[4];
    double* cc_t; int32_t* cc_n;
    // parameter-dependent condition / additive parameter affect (test/Callbacks2/continuous_callbacks.jl:317-345): the level is
    // cc_level + cc_lcoef * p[cc_lparam] (cc_lparam < 0: none); u[cc_acomp] += cc_acoef * p[cc_aparam] after the affine part
    // and the non-linear affect u[cc_qcomp] <- cc_qcoef * u[cc_qcomp]^2 (:222-250) in place of that component's affine map
    int32_t cc_lparam, cc_acomp, cc_aparam, cc_qcomp; double cc_lcoef, cc_acoef, cc_qcoef;
    double A[7][6];         // Tsit5 tableau (row 6 = b)
    double C[7];
    double BT[7];           // embedded error weights b - bhat
    double R[7][4];         // dense-output polynomials: b_j(theta) = sum_m R[j][m] theta^(m+1)
    // family events (VectorContinuousCallback, b200adj_set_family_events): the continuous callback's conditions and affect are
    // the ones compiled into the family struct (Fam::NC, condition, condition_grad, affect, affect_vjp; family_plugin.inc).
    // fe_nc > 0 selects them; fe_dir[c] is the direction of condition c (-1 down, +1 up, 0 both).  The forward kernel stores
    // with each event time of cc_t its event word cc_ev[cc_maxev][N]: bit 2c = condition c fired, bit 2c + 1 = it crossed upwards.
    int32_t fe_nc, fe_dir[8];
    int32_t* cc_ev;
};

// a family struct carries conditions and an affect (family_plugin.inc specialises this for B200ADJ_FAMILY_HAS_EVENTS)
template <class Fam> struct FamilyEvents { static constexpr bool value = false; };
__host__ __device__ constexpr uint32_t fe_fired(uint32_t word, int c) { return (word >> (2 * c)) & 1u; }
__host__ __device__ constexpr uint32_t fe_upward(uint32_t word, int c) { return (word >> (2 * c + 1)) & 1u; }

__device__ __forceinline__ void t5_weights(const T5aArgs& a, double th, double* w) {
#pragma unroll
    for (int j = 0; j < 7; j++) w[j] = th * (a.R[j][0] + th * (a.R[j][1] + th * (a.R[j][2] + th * a.R[j][3])));
}

// parameters in force after the first `upto` events (p0 = the caller's parameters of this member)
template <int P>
__device__ __forceinline__ void t5_event_params(const T5aArgs& a, int upto, const double* p0, double* p) {
#pragma unroll
    for (int q = 0; q < P; q++) p[q] = p0[q];
    if (!a.ev_ps) return;
    for (int e = 0; e < upto; e++) {
#pragma unroll
        for (int q = 0; q < P; q++) p[q] = a.ev_ps[e * P + q] * p[q] + a.ev_pc[e * P + q];
    }
}

template <int D> __host__ __device__ constexpr int t5_rec() { return 8 * D + 4; }      // doubles per record: a multiple of 4 (bulk copies move multiples of 16 B)
// pitch of the per-thread record buffers in shared memory: 16 B aligned (bulk-copy destination) with pitch / 2 odd, so that the
// 16 lanes of a half warp reading the same element hit 8 distinct 8-byte banks (2-way conflict; the unpadded pitch gives 4-way)
template <int D> __host__ __device__ constexpr int t5_pitch() { return 8 * D + 6; }

// bulk-copy helpers beside those of ode_tsit5.cuh (SASS: UBLKCP.S.G / UBLKCP.G.S)
__device__ __forceinline__ void fence_proxy_async_smem() { asm volatile("fence.proxy.async.shared::cta;" ::: "memory"); }
__device__ __forceinline__ void tma_store_1d(void* dst_gmem, const void* src_smem, uint32_t bytes) {
    asm volatile("cp.async.bulk.global.shared::cta.bulk_group [%0], [%1], %2;" ::"l"(dst_gmem), "r"(smem_u32(src_smem)), "r"(bytes) : "memory");
}
__device__ __forceinline__ void tma_store_commit() { asm volatile("cp.async.bulk.commit_group;" ::: "memory"); }
__device__ __forceinline__ void tma_store_wait_read() { asm volatile("cp.async.bulk.wait_group.read 0;" ::: "memory"); }
__device__ __forceinline__ void tma_store_wait_all() { asm volatile("cp.async.bulk.wait_group 0;" ::: "memory"); }

// Forward dense solution of one member, as the reverse solve sees it.  The solve runs downwards and evaluates the interpolant
// 6-9 times per step, mostly inside ONE forward interval.  Every lane of a warp has its own step sequence, so per-element
// loads would touch one cache line per lane and instruction (the first version of this kernel was bound by exactly that: the
// L1 tag stage, 37 k cycles per step and warp on the C1 ensemble).  Instead each THREAD owns two record buffers in shared
// memory and one mbarrier: entering interval iv it asks the TMA engine for the record of interval iv - 1 (one bulk copy of
// 8 D + 4 doubles); when the solve crosses the knot the record is there and the buffers swap.  Global memory is waited for
// only at the start and after a jump over several intervals.
template <int D>
struct T5Dense {
    static constexpr int REC = t5_rec<D>();
    const T5aArgs& a;
    const double* recs; const double* knots; int n;      // this member's records [n + 1][REC] and knots [n + 1]
    double* sc; int bs; uint64_t* bar;                   // this thread's two record buffers (sc, sc + bs) and its mbarrier (shared memory)
    mutable int cur = 0;
    mutable int cb = 0, civ = -1, aiv = -1;              // current buffer, its interval, the interval requested into the other one
    mutable uint32_t ph = 0;                             // parity of the mbarrier phase the next wait completes
    mutable double cta = 0.0, ctb = 0.0;
    __device__ __forceinline__ double T(int idx) const { return knots[idx]; }
    __device__ __forceinline__ const double* record(int idx) const { return recs + (int64_t)idx * REC; }
    __device__ __forceinline__ bool holds(int iv, double ta, double tb, double t, bool right) const {
        // interval iv = [ta, tb] is where the cursor search stops at once
        return right ? ((iv == 0 || ta <= t) && (iv == n - 1 || tb > t)) : ((iv == 0 || ta < t) && (iv == n - 1 || tb >= t));
    }
    __device__ __forceinline__ void request(int buf, int iv) const {
        // (no proxy fence: the buffer was only READ through the generic proxy, and those reads have returned their values --
        //  the same consumer-release -> producer-load order TMA pipelines rely on)
        mbar_expect_tx(bar, (uint32_t)(REC * sizeof(double)));
        tma_load_1d(sc + buf * bs, record(iv), (uint32_t)(REC * sizeof(double)), bar);
    }
    __device__ __forceinline__ void arrived() const { mbar_wait(bar, ph); ph ^= 1u; }
    // The records carry the interpolant in powers of theta (written so by the forward kernel):
    //   y(theta) = u_n + h theta (c0 + theta (c1 + theta (c2 + theta c3)))
    __device__ __forceinline__ void eval(double t, bool right, double* y) const {
        if (!(civ >= 0 && holds(civ, cta, ctb, t, right))) {
            bool got = false;
            if (aiv >= 0) {                               // the interval below was requested when this one was entered
                arrived();
                const double ata = sc[(cb ^ 1) * bs + 8 * D];
                if (holds(aiv, ata, cta, t, right)) { cb ^= 1; civ = aiv; ctb = cta; cta = ata; cur = civ; got = true; }
            }
            if (!got) {
                // cursor instead of a bisection over the knots: the adjoint solve visits the forward solution monotonically
                int iv = cur < n - 1 ? cur : n - 1;
                if (iv < 0) iv = 0;
                if (right) { while (iv > 0 && T(iv) > t) iv--; while (iv < n - 1 && T(iv + 1) <= t) iv++; }
                else { while (iv > 0 && T(iv) >= t) iv--; while (iv < n - 1 && T(iv + 1) < t) iv++; }
                cur = iv; civ = iv;
                request(cb, iv);
                arrived();
                cta = sc[cb * bs + 8 * D]; ctb = sc[cb * bs + 8 * D + 3];
            }
            aiv = civ - 1;
            if (aiv >= 0) request(cb ^ 1, aiv);
        }
        const double* b = sc + cb * bs;
        const double h = ctb - cta;
        const double th = (h == 0.0) ? 1.0 : (t - cta) * b[8 * D + 2];       // the record carries 1 / h
        const double g = h * th;
#pragma unroll
        for (int j = 0; j < D; j++)
            y[j] = fma(g, fma(th, fma(th, fma(th, b[D + 3 * D + j], b[D + 2 * D + j]), b[D + D + j]), b[D + j]), b[j]);
    }
};

// one Tsit5 step of length h from (t, z) with k[0] = rhs(t, z) given; fills k[1..6], znew
template <int L, class RHS>
__device__ __forceinline__ void t5_step(const T5aArgs& a, const RHS& rhs, double t, double h, const double* z, double (*k)[L], double* zn) {
    double tmp[L];
#pragma unroll
    for (int s = 1; s < 7; s++) {
#pragma unroll
        for (int c = 0; c < L; c++) {
            double acc = 0.0;
#pragma unroll
            for (int j = 0; j < 6; j++) if (j < s) acc += a.A[s][j] * k[j][c];
            tmp[c] = z[c] + h * acc;
        }
        if (s == 6) {
#pragma unroll
            for (int c = 0; c < L; c++) zn[c] = tmp[c];
        }
        rhs(t + a.C[s] * h, tmp, k[s]);
    }
}
template <int L>
__device__ __forceinline__ double t5_error(const T5aArgs& a, double h, const double* z, const double* zn, const double (*k)[L]) {
    double e2 = 0;
#pragma unroll
    for (int c = 0; c < L; c++) {
        double e = 0;
#pragma unroll
        for (int j = 0; j < 7; j++) e += a.BT[j] * k[j][c];
        e *= h;
        const double sc = a.abstol + a.reltol * fmax(fabs(z[c]), fabs(zn[c]));
        e2 += (e / sc) * (e / sc);
    }
    return sqrt(e2 / L);
}

// effective affine affect of the state-dependent event for a member with parameters p (constant along the solve)
template <int D, int P>
__device__ __forceinline__ void t5_cc_affect(const T5aArgs& a, const double* p, double* sc, double* sh) {
    double pv = 0.0;
#pragma unroll
    for (int q = 0; q < P; q++) if (q == a.cc_pparam) pv = p[q];
#pragma unroll
    for (int j = 0; j < D; j++) {
        const bool pc = (j == a.cc_pcomp);
        sc[j] = pc ? a.cc_psign * pv : a.cc_scale[j];
        sh[j] = pc ? 0.0 : a.cc_shift[j];
    }
    if (a.cc_acomp >= 0) {           // u[acomp] += acoef * p[aparam]
        double pa = 0.0;
#pragma unroll
        for (int q = 0; q < P; q++) if (q == a.cc_aparam) pa = p[q];
#pragma unroll
        for (int j = 0; j < D; j++) if (j == a.cc_acomp) sh[j] += a.cc_acoef * pa;
    }
}
// level of the condition u[cc_idx] - level: cc_level + cc_lcoef * p[cc_lparam]
template <int P>
__device__ __forceinline__ double t5_cc_level(const T5aArgs& a, const double* p) {
    double lv = a.cc_level;
    if (a.cc_lparam >= 0) {
#pragma unroll
        for (int q = 0; q < P; q++) if (q == a.cc_lparam) lv += a.cc_lcoef * p[q];
    }
    return lv;
}
template <int D>
__device__ __forceinline__ double t5_pick(const double* v, int idx) {
    double r = 0.0;
#pragma unroll
    for (int j = 0; j < D; j++) if (j == idx) r = v[j];
    return r;
}

// Condition policy of the state-dependent event: NC conditions g_c(y, p, t), each with its direction -- here the conditions
// compiled into the family (b200adj_set_family_events).  (The named condition u[cc_idx] - level keeps its own scalar loop in
// t5a_forward_kernel: routed through t5_find_event it compiles to different SASS, and its kernels are pinned.)
template <class Fam>
struct T5FamilyCond {
    static constexpr int NC = Fam::NC;
    const T5aArgs& a;
    __device__ __forceinline__ void operator()(const double* y, const double* p, double t, double* g) const { Fam::condition(y, p, t, g); }
    __device__ __forceinline__ int dir(int c) const { return a.fe_dir[c]; }
};

// Event search on one accepted step [t, t + h] (k1..k7 in registers, un = the end point): the conditions are evaluated on the
// dense output y(theta) at theta = j / 10 (interp_points = 10 of ContinuousCallback: a long step may hold a whole flight);
// the first sample interval in which any condition changes sign in its direction holds the event.  Every condition that
// crosses there is bisected to the last bit; theta* is the smallest root and the conditions whose root has the same bits
// fire together.  Conditions in `skip` (those that fired at the event the step starts on, ~0 with a random sign) take their
// side from the first sample instead.  Returns the event word (bit 2c fired, bit 2c + 1 upwards; 0 = no event) and theta*;
// *pending gets the same bits for the conditions that cross in that interval but whose roots have other bits
// (t5_fire_reached decides them once the step is redone).
template <int D, class Cond>
__device__ __forceinline__ uint32_t t5_find_event(const T5aArgs& a, const Cond& cond, const double* u, const double* un,
                                                  const double (*k)[D], const double* p, double t, double h, uint32_t skip, double* thstar,
                                                  uint32_t* pending) {
    constexpr int NC = Cond::NC;
    auto conds_at = [&](double th, double* g) {         // the full dense output y(theta), once per sample
        double y[D], w[7];
        t5_weights(a, th, w);
#pragma unroll
        for (int j = 0; j < D; j++) {
            double acc = 0.0;
#pragma unroll
            for (int s = 0; s < 7; s++) acc += w[s] * k[s][j];
            y[j] = u[j] + h * acc;
        }
        cond(y, p, t + th * h, g);
    };
    double gprev[NC], gj[NC], thprev = 0.0, lo = 0.0, hi = 1.0;
    cond(u, p, t, gprev);
    uint32_t cross = 0;
    for (int j = 1; j <= 10 && !cross; j++) {
        const double th = j == 10 ? 1.0 : 0.1 * j;
        if (j == 10) cond(un, p, t + h, gj); else conds_at(th, gj);
#pragma unroll
        for (int c = 0; c < NC; c++) {
            if (j == 1 && ((skip >> c) & 1u)) continue;
            const int dr = cond.dir(c);
            if ((dr <= 0 && gprev[c] > 0 && gj[c] <= 0) || (dr >= 0 && gprev[c] < 0 && gj[c] >= 0)) cross |= 1u << c;
        }
        if (cross) { lo = thprev; hi = th; }
        else {
#pragma unroll
            for (int c = 0; c < NC; c++) gprev[c] = gj[c];
            thprev = th;
        }
    }
    if (!cross) return 0u;
    double root[NC], ts = 2.0;
    bool any = false;
#pragma unroll
    for (int c = 0; c < NC; c++) {
        root[c] = 2.0;
        if (NC > 1 && !((cross >> c) & 1u)) continue;
        // bisection to the last bit; the root is the first theta on the far side
        const bool pos = gprev[c] > 0;
        double l = lo, r = hi;
        for (int it = 0; it < 200; it++) {
            const double mid = 0.5 * (l + r);
            if (!(mid > l && mid < r)) break;
            double gm[NC];
            conds_at(mid, gm);
            if ((gm[c] > 0) == pos && gm[c] != 0) l = mid; else r = mid;
        }
        root[c] = r;
        ts = any ? fmin(ts, r) : r;
        any = true;
    }
    uint32_t word = 0, pend = 0;
#pragma unroll
    for (int c = 0; c < NC; c++) {
        const uint32_t bits = (1u << (2 * c)) | ((gprev[c] < 0 ? 1u : 0u) << (2 * c + 1));
        if (root[c] == ts) word |= bits;
        else if ((cross >> c) & 1u) pend |= bits;
    }
    *thstar = ts;
    *pending = pend;
    return word;
}

// The conditions of `pending` whose value at the end point un of the redone step (time tn) has reached their far side or
// zero fire with the event.  The next step starts from un, and a condition that starts there on its far side or on zero can
// never satisfy the crossing test: a root a few ulps after theta* would otherwise be lost (its affect silently skipped).
template <class Fam>
__device__ __forceinline__ uint32_t t5_fire_reached(const double* un, const double* p, double tn, uint32_t pending) {
    if (!pending) return 0u;
    double g[Fam::NC];
    Fam::condition(un, p, tn, g);
    uint32_t word = 0;
#pragma unroll
    for (int c = 0; c < Fam::NC; c++)
        if (fe_fired(pending, c) && (fe_upward(pending, c) ? g[c] >= 0 : g[c] <= 0)) word |= pending & (3u << (2 * c));
    return word;
}

// CC: state-dependent event; FE (with CC): its conditions and affect are those of the family (T5FamilyCond), else named
template <class Fam, bool SHARED_P, bool CC = false, bool FE = false>
__global__ void __launch_bounds__(256) t5a_forward_kernel(const __grid_constant__ T5aArgs a) {
    constexpr int D = Fam::D, P = Fam::P;
    const int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= a.N) return;
    const int64_t N = a.N;
    double p[P];
#pragma unroll
    for (int q = 0; q < P; q++) p[q] = SHARED_P ? a.p[q] : a.p[(int64_t)q * N + i];
    constexpr int REC = t5_rec<D>();
    extern __shared__ __align__(16) double s_t5_stage[];     // [blockDim.x][t5_pitch]: the record of the step this thread has just accepted
    double* st = s_t5_stage + (size_t)threadIdx.x * t5_pitch<D>();
    double* recs = a.frecT + (int64_t)i * (a.maxs + 1) * REC;
    double* knots = a.ftT + (int64_t)i * (a.maxs + 1);
    double u[D], un[D], k[7][D];
#pragma unroll
    for (int j = 0; j < D; j++) u[j] = a.u0[(int64_t)j * N + i];
    knots[0] = a.t0;
    auto rhs = [&](double, const double* x, double* dx) { Fam::f(x, p, dx); };
    Fam::f(u, p, k[0]);
    double t = a.t0, h = a.dt0 > 0 ? a.dt0 : 1e-3 * (a.t1 - a.t0), qold = 1e-4;
    int n = 0, ksave = 0, stat = 0;
    long iters = 0;
    while (a.saved && ksave < a.K && a.saveat[ksave] <= a.t0) {
#pragma unroll
        for (int j = 0; j < D; j++) a.saved[((int64_t)ksave * D + j) * N + i] = u[j];
        ksave++;
    }
    int ev = 0;                                   // next event ahead of t (event times are tstops of the forward solve)
    const bool fixed = (a.flags & KF_FIXED_DT) != 0;      // constant step dt0, no error control (fixed-step Tsit5 with off-grid save times)
    bool after_event = false;                     // CC: the step starts on an event (condition ~0 with a random sign)
    int nfound = 0;
    const double cc_lev = (CC && !FE) ? t5_cc_level<P>(a, p) : 0.0;
    uint32_t fe_skip = 0, fe_word = 0;            // FE: conditions that fired at the event the step starts on; the event word
    // component cc_idx of the step's dense output at theta (k1..k7 in registers)
    auto cond_at = [&](double th, double hh) {
        double w[7];
        t5_weights(a, th, w);
        double r = 0.0;
#pragma unroll
        for (int j = 0; j < D; j++) {
            double acc = 0.0;
#pragma unroll
            for (int s = 0; s < 7; s++) acc += w[s] * k[s][j];
            if (j == a.cc_idx) r = u[j] + hh * acc;
        }
        return r - cc_lev;
    };
    while (t < a.t1) {
        if (++iters > 10000000L || n >= a.maxs) { stat = 2; break; }
        bool last = false;
        const double tend = (!CC && ev < a.nev) ? a.ev_t[ev] : a.t1;
        if (t + h >= tend || fabs(t + h - tend) < 100 * 2.22e-16 * fabs(tend)) { h = tend - t; last = true; }
        t5_step<D>(a, rhs, t, h, u, k, un);
        const double EEst = fixed ? 0.0 : t5_error<D>(a, h, u, un, k);
        if (!isfinite(EEst)) {                    // a trial step that overflowed: shrink (OrdinaryDiffEq does), give up below dtmin
            h *= 0.25;
            if (!(fabs(h) > 1e-14 * fmax(fabs(t), fabs(a.t1 - a.t0)))) { stat = 1; break; }
            continue;
        }
        const double q11 = pow(fmax(EEst, 1e-300), 7.0 / 50.0);
        double q = q11 / pow(qold, 2.0 / 25.0);
        q = fmax(1.0 / 10.0, fmin(5.0, q / 0.9));
        if (EEst <= 1.0) {
            double tn = last ? tend : t + h;
            bool at_event = !CC && last && ev < a.nev;
            if constexpr (FE) {
                // the family's conditions (t5_find_event): right after an event the conditions that fired there take their
                // side from the first sample; the step is redone up to theta* as below
                double thstar = 1.0;
                uint32_t pend = 0;
                uint32_t word = t5_find_event<D>(a, T5FamilyCond<Fam>{a}, u, un, k, p, t, h, fe_skip, &thstar, &pend);
                fe_skip = 0;
                if (word) {
                    // an event never lands on the time of the one before (a root a few ulps into the step, right after an
                    // event): the reverse pass tells events and their dense intervals apart by their times
                    double hh = thstar * h;
                    if (!(t + hh > t)) hh = fmax(fabs(t), 1e-300) * 2.220446049250313e-16;      // >= one ulp of t
                    t5_step<D>(a, rhs, t, hh, u, k, un);
                    tn = t + hh;
                    word |= t5_fire_reached<Fam>(un, p, tn, pend);
                    at_event = true;
                    if (nfound >= a.cc_maxev) { stat = 3; break; }
                    a.cc_t[(int64_t)nfound * N + i] = tn;
                    a.cc_ev[(int64_t)nfound * N + i] = (int32_t)word;
                    fe_word = word;
                    nfound++;
                }
            } else if (CC) {
                // sign changes of the condition on the dense output, sampled at theta = j / 10 (interp_points = 10 of
                // ContinuousCallback: a long step may hold a whole flight); right after an event the first sample decides the side
                double gprev = t5_pick<D>(u, a.cc_idx) - cc_lev, thprev = 0.0, lo = 0.0, hi = 1.0;
                bool hit = false;
                for (int j = 1; j <= 10 && !hit; j++) {
                    const double th = j == 10 ? 1.0 : 0.1 * j;
                    const double gj = (j == 10) ? t5_pick<D>(un, a.cc_idx) - cc_lev : cond_at(th, h);
                    if (after_event && j == 1) { gprev = gj; thprev = th; continue; }
                    if ((a.cc_dir <= 0 && gprev > 0 && gj <= 0) || (a.cc_dir >= 0 && gprev < 0 && gj >= 0)) { hit = true; lo = thprev; hi = th; }
                    else { gprev = gj; thprev = th; }
                }
                after_event = false;
                if (hit) {
                    // bisection of the crossing to the last bit, then the step is REDONE with h' = theta* h so that the stored
                    // dense data belong to [t, tau] (k[0] = f(u) is still valid)
                    const bool pos = gprev > 0;
                    for (int it = 0; it < 200; it++) {
                        const double mid = 0.5 * (lo + hi);
                        if (!(mid > lo && mid < hi)) break;
                        const double gm = cond_at(mid, h);
                        if ((gm > 0) == pos && gm != 0) lo = mid; else hi = mid;
                    }
                    const double hh = hi * h;
                    t5_step<D>(a, rhs, t, hh, u, k, un);
                    tn = t + hh;
                    at_event = true;
                    if (nfound >= a.cc_maxev) { stat = 3; break; }
                    a.cc_t[(int64_t)nfound * N + i] = tn;
                    nfound++;
                }
            }
            // a save time that coincides with an event records the post-event state (saved after the affect, below)
            while (a.saved && ksave < a.K && (a.saveat[ksave] < tn || (a.saveat[ksave] == tn && !at_event))) {
                const double hh = tn - t, th = (hh == 0.0) ? 1.0 : (a.saveat[ksave] - t) / hh;
                double w[7];
                t5_weights(a, th, w);
#pragma unroll
                for (int j = 0; j < D; j++) {
                    double acc = 0.0;
#pragma unroll
                    for (int s = 0; s < 7; s++) acc += w[s] * k[s][j];
                    a.saved[((int64_t)ksave * D + j) * N + i] = u[j] + hh * acc;
                }
                ksave++;
            }
            {   // the step's record (start state, k1..k7, knots): staged in shared memory, then ONE bulk store to this member's row
                tma_store_wait_read();                                 // the previous record has left the staging buffer
#pragma unroll
                for (int j = 0; j < D; j++) st[j] = u[j];
                // the stages enter the record as the coefficients of the interpolant in powers of theta,
                //   y(theta) = u_n + h theta (c0 + theta (c1 + theta (c2 + theta c3))),  c_m = sum_s R[s][m] k_s
                // (b_s(theta) = sum_m R[s][m] theta^(m+1)): computed once here, every lookup of the reverse solve and of the
                // quadrature is then 4 FMAs per component instead of the seven weights + a 7-term combination
#pragma unroll
                for (int j = 0; j < D; j++) {
#pragma unroll
                    for (int m = 0; m < 4; m++) {
                        double c = 0.0;
#pragma unroll
                        for (int s = 0; s < 7; s++) c += a.R[s][m] * k[s][j];
                        st[D + m * D + j] = c;
                    }
#pragma unroll
                    for (int m = 4; m < 7; m++) st[D + m * D + j] = 0.0;
                }
                const double hrec = tn - t;
                st[8 * D] = t; st[8 * D + 1] = hrec; st[8 * D + 2] = 1.0 / hrec; st[8 * D + 3] = tn;
                fence_proxy_async_smem();
                tma_store_1d(recs + (int64_t)n * REC, st, (uint32_t)(REC * sizeof(double)));
                tma_store_commit();
            }
            if (at_event) {
                // affect!: the next step starts from the post-event state; k7 = f(u^-) stays with the step just stored
                if constexpr (FE) {
                    // affect!(integrator, ev) of the family: ev[c] = +1 / -1 for a condition that crossed upwards / downwards
                    int evs[Fam::NC];
                    double up[D];
#pragma unroll
                    for (int c = 0; c < Fam::NC; c++) evs[c] = fe_fired(fe_word, c) ? (fe_upward(fe_word, c) ? 1 : -1) : 0;
                    Fam::affect(evs, un, p, up);
#pragma unroll
                    for (int j = 0; j < D; j++) un[j] = up[j];
                    fe_skip = 0;
#pragma unroll
                    for (int c = 0; c < Fam::NC; c++) fe_skip |= fe_fired(fe_word, c) << c;
                } else if (CC) {
                    double sc[D], sh[D];
                    t5_cc_affect<D, P>(a, p, sc, sh);
#pragma unroll
                    for (int j = 0; j < D; j++) un[j] = (j == a.cc_qcomp) ? a.cc_qcoef * un[j] * un[j] : sc[j] * un[j] + sh[j];
                    after_event = true;
                } else {
#pragma unroll
                for (int j = 0; j < D; j++) un[j] = a.ev_s[ev * D + j] * un[j] + a.ev_c[ev * D + j];
                if (a.ev_ac) {
                    const int ac = a.ev_ac[ev], ak = a.ev_ak[ev];
                    double pa = 0.0;
#pragma unroll
                    for (int q = 0; q < P; q++) if (q == ak) pa = p[q];
#pragma unroll
                    for (int j = 0; j < D; j++) if (j == ac) un[j] += a.ev_af[ev] * pa;
                }
                if (a.ev_ps) {
#pragma unroll
                    for (int q = 0; q < P; q++) p[q] = a.ev_ps[ev * P + q] * p[q] + a.ev_pc[ev * P + q];
                }
                ev++;
                }
                Fam::f(un, p, k[6]);
                while (a.saved && ksave < a.K && a.saveat[ksave] == tn) {
#pragma unroll
                    for (int j = 0; j < D; j++) a.saved[((int64_t)ksave * D + j) * N + i] = un[j];
                    ksave++;
                }
            }
#pragma unroll
            for (int j = 0; j < D; j++) { u[j] = un[j]; k[0][j] = k[6][j]; }
            t = tn; knots[n + 1] = t;
            n++;
            qold = fmax(EEst, 1e-4);
            h = fixed ? a.dt0 : h / q;            // constant step: back to dt after a step clipped at an event (dtcache)
        } else {
            h = h / fmin(5.0, q11 / 0.9);
        }
    }
    a.fn[i] = n;
    {   // the terminal record: final state and time
        tma_store_wait_read();
#pragma unroll
        for (int j = 0; j < D; j++) st[j] = u[j];
#pragma unroll
        for (int c = D; c < REC; c++) st[c] = 0.0;
        st[8 * D] = t; st[8 * D + 3] = t;
        fence_proxy_async_smem();
        tma_store_1d(recs + (int64_t)n * REC, st, (uint32_t)(REC * sizeof(double)));
        tma_store_commit();
        tma_store_wait_all();
    }
    if (CC) a.cc_n[i] = nfound;
    bool ok = true;
#pragma unroll
    for (int j = 0; j < D; j++) ok = ok && isfinite(u[j]);
    if (!ok && stat == 0) stat = 1;
    if (a.status) a.status[i] = stat;
}

// reverse adjoint solve.  SA_INTERP: z = [lambda; mu] (L = D + P); SA_GAUSS / SA_QUAD: z = lambda (L = D);
// SA_BACKSOLVE: z = [lambda; mu; y] (L = 2D + P), y integrated backwards and reset from the forward solution at the
// checkpoints (every forward knot = sol.t, the direct-interface default, or the save times), which are tstops of the reverse
// solve (src/backsolve_adjoint.jl:32-61, :523-546; src/sensitivity_interface.jl:433, :484-486; the reference's own
// Lorenz check, test/Core3/adjoint.jl:1157-1241)
// (A register cap -- __maxnreg__(144): 14 warps per SM, the 65 536-member C1 shard in ONE wave instead of two -- was measured
// twice and rejected: 8.9 ms against 7.25 ms uncapped.  Block sizes 32 / 64 / 128 (8 to 11 resident warps per SM) all give
// 7.25 ms: the time is two rounds of a latency-bound per-warp chain, see DESIGN.md 4.4.)
template <class Fam, int SA, bool SHARED_P, int COST, bool CC = false, bool FE = false>
__global__ void __launch_bounds__(256) t5a_reverse_kernel(const __grid_constant__ T5aArgs a) {
    constexpr int D = Fam::D, P = Fam::P, L = (SA == SA_INTERP) ? D + P : (SA == SA_BACKSOLVE ? 2 * D + P : D);
    constexpr int YO = (SA == SA_BACKSOLVE) ? D + P : 0;          // offset of y inside z (Backsolve)
    const int64_t gi = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
    const bool active = gi < a.N;
    const int64_t i = active ? gi : a.N - 1;
    const int64_t N = a.N;
    double p[P], acc[P];
#pragma unroll
    for (int q = 0; q < P; q++) { p[q] = SHARED_P ? a.p[q] : a.p[(int64_t)q * N + i]; acc[q] = 0.0; }
    if (a.ev_ps) {                                 // the reverse solve starts on the last segment: parameters after all events
        double p0[P];
#pragma unroll
        for (int q = 0; q < P; q++) p0[q] = p[q];
        t5_event_params<P>(a, a.nev, p0, p);
    }
    constexpr int REC = t5_rec<D>();
    extern __shared__ __align__(16) double s_t5_dense[];     // [2][blockDim.x][t5_pitch] record buffers, then [blockDim.x] mbarriers
    const int bufstride = (int)blockDim.x * t5_pitch<D>();
    uint64_t* my_bar = reinterpret_cast<uint64_t*>(s_t5_dense + (size_t)2 * bufstride) + threadIdx.x;
    mbar_init(my_bar, 1);
    mbar_fence_init();
    T5Dense<D> sol{a, a.frecT + (int64_t)i * (a.maxs + 1) * REC, a.ftT + (int64_t)i * (a.maxs + 1), a.fn[i],
                   s_t5_dense + (size_t)threadIdx.x * t5_pitch<D>(), bufstride, my_bar};
    sol.cur = sol.n - 1;
    double z[L], zn[L], k[7][L];
#pragma unroll
    for (int c = 0; c < L; c++) z[c] = 0.0;
    double tev = INFINITY;                        // event time just crossed (y(tev) = left limit from there on)
    // adjoint RHS: dlam = -J(y(t))' lam, dmu = -F(y(t))' lam  (right-continuous forward lookup)
    auto rhs = [&](double tt, const double* x, double* dx) {
        double y[D];
        if (SA == SA_BACKSOLVE) {
#pragma unroll
            for (int j = 0; j < D; j++) y[j] = x[YO + j];          // y is part of the state
        } else sol.eval(tt, tt != tev, y);                         // the left limit at an event the solve has just crossed
        Fam::vjp_u(y, p, x, dx);
#pragma unroll
        for (int j = 0; j < D; j++) dx[j] = -dx[j];
        if (a.flags & KF_CONT_COST) {                                          // src/derivative_wrappers.jl:1411-1442
#pragma unroll
            for (int j = 0; j < D; j++) dx[j] -= a.cont_a[j] * y[j] + a.cont_b[j];
        }
        if (SA == SA_INTERP || SA == SA_BACKSOLVE) {
            double dg[P];
            Fam::vjp_p(y, p, x, dg);
#pragma unroll
            for (int q = 0; q < P; q++) dx[D + q] = -dg[q];
        }
        if (SA == SA_BACKSOLVE) Fam::f(y, p, dx + YO);            // dy/dt = f(y)
    };
    const double T = a.t1, t0 = a.t0;
    double t = T;
    // CC: this member's own event list, found by the forward solve
    auto evt = [&](int e) { return CC ? a.cc_t[(int64_t)e * N + i] : a.ev_t[e]; };
    int cur = a.K - 1, nrev = 0, ck = sol.n, evc = (CC ? a.cc_n[i] : a.nev) - 1;
    // a member whose forward solve stopped before t1 (status 1 / 2 / 3) has records only up to the break: NaN, as for a
    // reverse solve that overflows, not the gradient of a trajectory that was never solved
    bool fsal_ok = false, overflow = a.status[i] != 0;
    const bool ckpt_on = !(a.flags & KF_NO_CHECKPOINTING), every = (a.flags & KF_CKPT_EVERY_STEP);
    if (SA == SA_BACKSOLVE) {
#pragma unroll
        for (int j = 0; j < D; j++) z[YO + j] = sol.record(sol.n)[j];     // y(T) = sol.u[end]
    }
    // Backsolve checkpoint callback (runs before the loss jump, CallbackSet order): y <- sol(t) at a checkpoint
    auto ckpt_if_at = [&](double tt) {
        if (SA != SA_BACKSOLVE || !ckpt_on) return;
        const double tol = EPS100 * fmax(fabs(tt), 1.0);
        if (every) {
            while (ck >= 0 && sol.T(ck) > tt + tol) ck--;
            if (ck >= 0 && fabs(sol.T(ck) - tt) <= tol) {
#pragma unroll
                for (int j = 0; j < D; j++) z[YO + j] = sol.record(ck)[j];
                fsal_ok = false;
            }
        } else if (cur >= 0 && fabs(a.saveat[cur] - tt) <= tol) {
            double y[D];
            sol.eval(a.saveat[cur], evc >= 0 && evt(evc) == a.saveat[cur], y);      // post-event state at a coinciding event
#pragma unroll
            for (int j = 0; j < D; j++) z[YO + j] = y[j];
            fsal_ok = false;
        }
    };
    // reverse affect of a preset-time event: lam(tau-) = scale .* lam(tau+); Backsolve takes y(tau-) from the forward
    // solution (the reference keeps it as `uleft` of the TrackedAffect).  Runs after the checkpoint reset and the loss jump.
    auto event_if_at = [&](double tt) {
        while (evc >= 0 && fabs(evt(evc) - tt) <= EPS100 * fmax(fabs(tt), 1.0)) {
            if constexpr (FE) {
                // state-dependent event of the family's conditions and affect (the implicit event-time correction of
                // src/callback_tracking.jl:232-480): with u+ = a(u-, p), c = the lowest condition that fired, g_c(u-, p, tau) = 0,
                //   (mu_u, mu_p) = ((da/du)'lam+, (da/dp)'lam+),  den = dg/du . f(u-) + dg/dt,  w = mu_u . f(u-) - lam+ . f(u+)
                //   lam- = mu_u - dg/du (w / den),  dG/dp += mu_p - dg/dp (w / den)
                // For g = u_i - level - lcoef p_k and a diagonal affect this is the named formula of the branch below.
                constexpr int NC = Fam::NC;
                double um[D], up[D], fm[D], fp[D], mu[D], mp[P], gu[D], gp[P];
                const double tau = evt(evc);
                sol.eval(tau, false, um); sol.eval(tau, true, up);
                Fam::f(um, p, fm); Fam::f(up, p, fp);
                const uint32_t word = (uint32_t)a.cc_ev[(int64_t)evc * N + i];
                int evs[NC], cf = 0;
#pragma unroll
                for (int c = NC - 1; c >= 0; c--) {
                    evs[c] = fe_fired(word, c) ? (fe_upward(word, c) ? 1 : -1) : 0;
                    if (evs[c]) cf = c;
                }
                Fam::affect_vjp(evs, um, p, z, mu, mp);
                const double gt = Fam::condition_grad(cf, um, p, tau, gu, gp);
                double den = gt, w = 0.0;
#pragma unroll
                for (int j = 0; j < D; j++) { den += gu[j] * fm[j]; w += mu[j] * fm[j] - z[j] * fp[j]; }
                const double r = w / den;
#pragma unroll
                for (int q = 0; q < P; q++) {
                    const double dq = mp[q] - gp[q] * r;
                    if (SA == SA_INTERP || SA == SA_BACKSOLVE) z[D + (L > D ? q : 0)] += dq; else acc[q] += dq;
                }
#pragma unroll
                for (int j = 0; j < D; j++) z[j] = mu[j] - gu[j] * r;
                if (SA == SA_BACKSOLVE) {
#pragma unroll
                    for (int j = 0; j < D; j++) z[YO + j] = um[j];
                }
            } else if constexpr (CC) {
                // state-dependent event time (the implicit correction of src/callback_tracking.jl:232-480): with u+ = A u- + c,
                // g(u-) = 0:  lam- = A'lam+ - e_ci [(A f- - f+)'lam+] / f-[ci],   dG/dp += (dA/dp u-)'lam+
                double um[D], up[D], fm[D], fp[D], sc[D], sh[D];
                const double tau = evt(evc);
                sol.eval(tau, false, um); sol.eval(tau, true, up);
                Fam::f(um, p, fm); Fam::f(up, p, fp);
                t5_cc_affect<D, P>(a, p, sc, sh);
                if (a.cc_qcomp >= 0) {       // u_q <- qcoef u_q^2: the Jacobian 2 qcoef u_q- takes the place of the scale
#pragma unroll
                    for (int j = 0; j < D; j++) if (j == a.cc_qcomp) sc[j] = 2.0 * a.cc_qcoef * um[j];
                }
                double wl = 0.0;
#pragma unroll
                for (int j = 0; j < D; j++) wl += (sc[j] * fm[j] - fp[j]) * z[j];
                if (a.cc_pcomp >= 0) {
                    const double gpar = a.cc_psign * t5_pick<D>(um, a.cc_pcomp) * t5_pick<D>(z, a.cc_pcomp);
#pragma unroll
                    for (int q = 0; q < P; q++) if (q == a.cc_pparam) {
                        if (SA == SA_INTERP || SA == SA_BACKSOLVE) z[D + (L > D ? q : 0)] += gpar; else acc[q] += gpar;
                    }
                }
                const double corr = wl / t5_pick<D>(fm, a.cc_idx);
                if (a.cc_acomp >= 0) {       // u+[acomp] += acoef p[aparam]: (da/dp)'lam+
                    const double gadd = a.cc_acoef * t5_pick<D>(z, a.cc_acomp);
#pragma unroll
                    for (int q = 0; q < P; q++) if (q == a.cc_aparam) {
                        if (SA == SA_INTERP || SA == SA_BACKSOLVE) z[D + (L > D ? q : 0)] += gadd; else acc[q] += gadd;
                    }
                }
                if (a.cc_lparam >= 0) {      // g = u_i - level - lcoef p[lparam]: -(dg/dp) w / (dg/du . f-)
                    const double glev = a.cc_lcoef * corr;
#pragma unroll
                    for (int q = 0; q < P; q++) if (q == a.cc_lparam) {
                        if (SA == SA_INTERP || SA == SA_BACKSOLVE) z[D + (L > D ? q : 0)] += glev; else acc[q] += glev;
                    }
                }
#pragma unroll
                for (int j = 0; j < D; j++) { z[j] *= sc[j]; if (j == a.cc_idx) z[j] -= corr; }
                if (SA == SA_BACKSOLVE) {
#pragma unroll
                    for (int j = 0; j < D; j++) z[YO + j] = um[j];
                }
            } else {
            double gadd = 0.0;        // (da/dp)'lam+ of u[ac] += af p[ak], taken before lam is scaled
            if (a.ev_ac) gadd = a.ev_af[evc] * t5_pick<D>(z, a.ev_ac[evc]);
#pragma unroll
            for (int j = 0; j < D; j++) z[j] *= a.ev_s[evc * D + j];
            if (SA == SA_BACKSOLVE) {
                double y[D];
                sol.eval(evt(evc), false, y);
#pragma unroll
                for (int j = 0; j < D; j++) z[YO + j] = y[j];
            }
            if (a.ev_ps) {
                // p+ = s_p .* p- + c_p: dG/dp- = s_p .* dG/dp+ (+ what accumulates below tau with p-); parameters of the
                // segment below re-derived from the caller's p
#pragma unroll
                for (int q = 0; q < P; q++) {
                    if (SA == SA_INTERP || SA == SA_BACKSOLVE) z[D + (L > D ? q : 0)] *= a.ev_ps[evc * P + q];
                    else acc[q] *= a.ev_ps[evc * P + q];
                }
                double p0[P];
#pragma unroll
                for (int q = 0; q < P; q++) p0[q] = SHARED_P ? a.p[q] : a.p[(int64_t)q * N + i];
                t5_event_params<P>(a, evc, p0, p);
            }
            if (a.ev_ac) {            // with respect to the parameters in force before the event
                const int ak = a.ev_ac[evc] >= 0 ? a.ev_ak[evc] : -1;
#pragma unroll
                for (int q = 0; q < P; q++) if (q == ak) {
                    if (SA == SA_INTERP || SA == SA_BACKSOLVE) z[D + (L > D ? q : 0)] += gadd; else acc[q] += gadd;
                }
            }
            }
            tev = tt; evc--; fsal_ok = false;
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
                    } else
                    sol.eval(a.saveat[cur], true, y);
#pragma unroll
                    for (int j = 0; j < D; j++) z[j] += a.cost_a[j] * y[j] + a.cost_b[j];
                }
            }
            cur--; fsal_ok = false;
        }
    };
    ckpt_if_at(t);
    jump_if_at(t);
    double h = a.dt0 > 0 ? -a.dt0 : -1e-4 * (T - t0), qold = 1e-4;
    const bool fixed = (a.flags & KF_FIXED_DT) != 0;
    long iters = 0;
    while (!overflow && t > t0 && sol.n > 0) {
        if (++iters > 50000000L || (SA == SA_QUAD && nrev >= a.maxs)) { overflow = true; break; }
        double tstop = t0;
        if (cur >= 0 && a.saveat[cur] < t && a.saveat[cur] > tstop) tstop = a.saveat[cur];
        if (evc >= 0 && evt(evc) < t && evt(evc) > tstop) tstop = evt(evc);
        if (SA == SA_BACKSOLVE && ckpt_on && every) {            // every forward knot is a tstop of the reverse solve
            int c2 = ck;
            while (c2 >= 0 && sol.T(c2) >= t - EPS100 * fmax(fabs(t), 1.0)) c2--;
            if (c2 >= 0 && sol.T(c2) > tstop) tstop = sol.T(c2);
        }
        double tn = tstop_snap(t + h, tstop);
        if (tn < tstop) tn = tstop;
        const double hs = tn - t;
        if (!fsal_ok) rhs(t, z, k[0]);
        t5_step<L>(a, rhs, t, hs, z, k, zn);
        const double EEst = fixed ? 0.0 : t5_error<L>(a, hs, z, zn, k);
        if (!isfinite(EEst)) {
            h = 0.25 * hs; fsal_ok = true;
            if (!(fabs(h) > 1e-14 * fmax(fabs(t), fabs(T - t0)))) { overflow = true; break; }
            continue;
        }
        const double q11 = pow(fmax(EEst, 1e-300), 7.0 / 50.0);
        const double q = fmax(0.1, fmin(5.0, q11 / pow(qold, 2.0 / 25.0) / 0.9));
        if (EEst > 1.0) { h = hs / fmin(5.0, q11 / 0.9); fsal_ok = true; continue; }
        qold = fmax(EEst, 1e-4); h = fixed ? -a.dt0 : hs / q;      // constant step: back to dt after a step clipped at a tstop
        if (SA == SA_GAUSS) {
            const double gx[3] = {-0.7745966692414834, 0.0, 0.7745966692414834};
            const double gw[3] = {0.5555555555555556, 0.8888888888888888, 0.5555555555555556};
#pragma unroll
            for (int g = 0; g < 3; g++) {
                const double tj = 0.5 * (tn - t) * gx[g] + 0.5 * (tn + t), th = (tj - t) / hs;
                double w[7], lq[D], y[D], dg[P];
                t5_weights(a, th, w);
#pragma unroll
                for (int j = 0; j < D; j++) {
                    double s_ = 0.0;
#pragma unroll
                    for (int s = 0; s < 7; s++) s_ += w[s] * k[s][j];
                    lq[j] = z[j] + hs * s_;
                }
                sol.eval(tj, false, y);
                Fam::vjp_p(y, p, lq, dg);
#pragma unroll
                for (int q2 = 0; q2 < P; q2++) acc[q2] += (0.5 * (tn - t)) * gw[g] * (-dg[q2]);
            }
        } else if (SA == SA_GK) {
            // GaussKronrodAdjoint: error-controlled G3/K7 quadrature of the accepted step (ros23.cuh::integrate_gk_step)
            auto node = [&](double tj, double* out) {
                const double th = (tj - t) / hs;
                double w[7], lq[D], y[D];
                t5_weights(a, th, w);
#pragma unroll
                for (int j = 0; j < D; j++) {
                    double s_ = 0.0;
#pragma unroll
                    for (int s = 0; s < 7; s++) s_ += w[s] * k[s][j];
                    lq[j] = z[j] + hs * s_;
                }
                sol.eval(tj, false, y);
                Fam::vjp_p(y, p, lq, out);
#pragma unroll
                for (int q2 = 0; q2 < P; q2++) out[q2] = -out[q2];
            };
            integrate_gk_step<P, 3>(node, t, tn, acc);
        } else if (SA == SA_QUAD && active) {
            double* rec = a.rrec + ((int64_t)i * a.maxs + nrev) * quad_pad(3 + 8 * D);
            rec[0] = t; rec[1] = hs; rec[2 + 8 * D] = 1.0 / hs;
            a.rend[(int64_t)i * a.maxs + nrev] = t + hs;
#pragma unroll
            for (int j = 0; j < D; j++) rec[2 + j] = z[j];
#pragma unroll
            for (int s = 0; s < 7; s++)
#pragma unroll
                for (int j = 0; j < D; j++) rec[2 + (1 + s) * D + j] = k[s][j];
        }
        nrev++;
#pragma unroll
        for (int c = 0; c < L; c++) { z[c] = zn[c]; k[0][c] = k[6][c]; }
        fsal_ok = true;
        t = tn;
        ckpt_if_at(t);
        jump_if_at(t);
        event_if_at(t);
    }
    const double qnan = __longlong_as_double(0x7ff8000000000000LL);
    if (active) {
#pragma unroll
        for (int j = 0; j < D; j++) a.du0[(int64_t)j * N + i] = overflow ? qnan : z[j];
        if (SA == SA_QUAD) a.rn[i] = overflow ? -1 : nrev;
    }
    if (SA != SA_QUAD) {
        double out[P];
#pragma unroll
        for (int q = 0; q < P; q++) out[q] = overflow ? qnan : ((SA == SA_INTERP || SA == SA_BACKSOLVE) ? z[(L > D ? D : 0) + (L > D ? q : 0)] : acc[q]);
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
}

// QuadratureAdjoint integrand on the two dense solutions (warp-cooperative lookups inside the segment's brackets, quadgk.cuh)
template <class Fam, int D, int P>
struct T5aQuadCtx {
    static constexpr int FWP = quad_pad(8 * D + 3), RWP = quad_pad(3 + 8 * D);
    const T5aArgs& a; const double* ftT; const double* frecT; const double* rrec; const double* rend;      // this member's rows
    int nf, nrev; double p[P];
    __device__ __forceinline__ bool valid() const { return nrev >= 0; }
    __device__ __forceinline__ bool empty() const { return nrev == 0; }
    __device__ __forceinline__ QuadBracket root() const { return QuadBracket{0, nf - 1, 0, nrev - 1}; }
    __device__ __forceinline__ void eval(double t, const QuadBracket& br, int lane, double* out, int* fiv, int* riv) const {
        double y[D], lam[D], w[7];
        const int iv = br.flo + coop_count<true>([&](int j) { return __ldg(ftT + j); }, br.flo + 1, br.fhi - br.flo, t, lane);
        const int lo = br.rlo + coop_count<false>([&](int j) { return __ldg(rend + j); }, br.rlo, br.rhi - br.rlo, t, lane);
        *fiv = iv; *riv = lo;
        {
            const double* r = frecT + iv * FWP;                  // (u[D], c0..c3[D] (powers of theta), -, t_a, h, 1/h)
            const double ta = __ldg(r + 8 * D), h = __ldg(r + 8 * D + 1);
            const double th = (h == 0.0) ? 1.0 : (t - ta) * __ldg(r + 8 * D + 2), g = h * th;
#pragma unroll
            for (int j = 0; j < D; j++)
                y[j] = fma(g, fma(th, fma(th, fma(th, __ldg(r + 4 * D + j), __ldg(r + 3 * D + j)), __ldg(r + 2 * D + j)), __ldg(r + D + j)), __ldg(r + j));
        }
        {
            const double* r = rrec + lo * RWP;                   // (t_start, h, z[D], k[7][D], 1/h)
            const double ts = __ldg(r), h = __ldg(r + 1);
            t5_weights(a, (t - ts) * __ldg(r + 2 + 8 * D), w);
#pragma unroll
            for (int j = 0; j < D; j++) {
                double s_ = 0.0;
#pragma unroll
                for (int s = 0; s < 7; s++) s_ += w[s] * __ldg(r + 2 + (1 + s) * D + j);
                lam[j] = __ldg(r + 2 + j) + h * s_;
            }
        }
        Fam::vjp_p(y, p, lam, out);
    }
};

template <class Fam, bool SHARED_P>
__global__ void __launch_bounds__(QUAD_WARPS * 32) t5a_quadrature_kernel(const __grid_constant__ T5aArgs a) {
    constexpr int D = Fam::D, P = Fam::P;
    extern __shared__ double s_quad_l1[];
    const int lane = threadIdx.x & 31;
    const int64_t N = a.N;
    double acc[P];
#pragma unroll
    for (int q = 0; q < P; q++) acc[q] = 0.0;
    auto make = [&](int64_t i) {
        T5aQuadCtx<Fam, D, P> c{a, a.ftT + (int64_t)i * (a.maxs + 1), a.frecT + (int64_t)i * (a.maxs + 1) * t5_rec<D>(),
                                a.rrec + (int64_t)i * a.maxs * quad_pad(3 + 8 * D), a.rend + (int64_t)i * a.maxs, a.fn[i], a.rn[i], {}};
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
