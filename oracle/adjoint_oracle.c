/*
 * oracle/adjoint_oracle.c  --  TEST INFRASTRUCTURE ONLY.
 *
 * CPU restatement (plain C, fp64, OpenMP over ensemble members) of the reverse-mode
 * continuous-adjoint hot path of SciML/SciMLSensitivity.jl v7.112.3.  It is the CHECKER
 * for the device kernels: only tests/, __graft_entry__.smoke() and bench.py's cpu_baseline /
 * --impl reference legs may load it.  The product path (libb200adj.so) never links or calls it.
 *
 * PARITY STATUS: pinned by the literal results the reference itself holds for this path, "parity unpinned"
 * at the bit level elsewhere.  The reference is pure Julia, Julia is not installed in this image, and the
 * reference ships no golden VECTORS for this path (SURVEY.md finding 5).  Reference-held numbers reproduced
 * (tests/test_reference_held_numbers.py): the printed optimum 0.866554105436901 of
 * docs/src/examples/hybrid_jump/bouncing_ball.md:60 as the root of the adjoint gradient (1e-14), the
 * first-impact fixture of test/Callbacks2/continuous_vs_discrete.jl:19-21 (4e-15), gND of
 * test/Callbacks2/continuous_callbacks.jl:343 at the reference's rtol 1e-10 (2e-15), the closed form of the
 * "Dosing example" (test/Callbacks1/discrete_callbacks.jl:401-427).  For the paths without a reference-held
 * literal (fixed-step Tsit5, Rosenbrock23, SDE) the oracle is pinned by the reference's own test RELATIONS
 * (tests/test_oracle_relations.py): cross-sensealg agreement (test/Core3/adjoint.jl:366-404),
 * agreement with differentiation through the solver (test/Core3/adjoint.jl:691-705),
 * du0 agreement (:865-908), Lorenz Backsolve==Interpolating (:1157-1241), closed-form linear SDE
 * gradients (test/SDE1/sde_stratonovich.jl:105-113), transformed drift value
 * (test/SDE3/sde_transformation_test.jl:25-38).
 *
 * Third-party arithmetic restated here (not vendored under /root/reference; SURVEY.md App. B):
 *   OrdinaryDiffEq  Tsit5 (tableau + 4th-order dense output), Rosenbrock23 (ode23s form),
 *   StochasticDiffEq EM / EulerHeun, DiffEqCallbacks IntegratingSumCallback (Gauss-Legendre per step),
 *   PresetTimeCallback (tstops + affect), QuadGK (adaptive G7/K15), DiffEqNoiseProcess reverse(W).
 *
 * What each block follows in the reference:
 *   adjoint RHS      src/interpolating_adjoint.jl:150-174, src/gauss_adjoint.jl:118-128,
 *                    src/quadrature_adjoint.jl:35-46, src/backsolve_adjoint.jl:32-61
 *   forward lookup   split_states -> sol(y,t,continuity=:right)  src/interpolating_adjoint.jl:190-205
 *   jumps            ReverseLossCallback  src/adjoint_common.jl:754-821 (lambda += dgdu at t_k, FSAL reset)
 *   Gauss integrand  src/gauss_adjoint.jl:745-759 and driver :766-870
 *   Quadrature       src/quadrature_adjoint.jl:486-508 (integrand), :510-633 (interval loop)
 *   Backsolve SDE    src/backsolve_adjoint.jl:274-419, :523-546, diag-noise VJP layout
 *                    src/derivative_wrappers.jl:1197-1199, Ito transform src/sde_tools.jl:29-66
 *   extraction       du0 = z[1:d], dp = z[d+1:d+P]'  src/sensitivity_interface.jl:500-508
 */
#include <math.h>
#include <stdint.h>
#include <stdlib.h>
#include <string.h>
#include <stdio.h>
#ifdef _OPENMP
#include <omp.h>
#endif

/* ---- enums: values shared (by convention, not by include) with include/b200adj.h ---- */
enum { FAM_LV = 0, FAM_LORENZ = 1, FAM_ROBERTSON = 2, FAM_SDE_LV = 3, FAM_MLP = 4, FAM_SDE_LINEAR = 5, FAM_BALL = 6, FAM_RELAX = 7 };
enum { SA_INTERPOLATING = 0, SA_GAUSS = 1, SA_QUADRATURE = 2, SA_BACKSOLVE = 3, SA_GAUSSKRONROD = 4 };
enum { ST_TSIT5_FIXED = 0, ST_ROSENBROCK23 = 1, ST_EM = 2, ST_EULER_HEUN = 3, ST_TSIT5_ADAPTIVE = 4 };
enum { COST_EXPLICIT = 0, COST_AFFINE = 1 };

typedef struct {
    int32_t family, sensealg, stepper, cost_kind;
    int32_t d, P, m, K;
    int64_t N;
    double t0, t1, dt, abstol, reltol;      /* forward (and adjoint) solver tolerances   */
    double quad_abstol, quad_reltol;        /* QuadratureAdjoint quadgk tolerances        */
    double cost_a, cost_b;                  /* COST_AFFINE: dLdu_k = a*u(t_k) + b         */
    int32_t shared_p;                       /* 1: p[P], dp[P] summed; 0: p[P][N], dp[P][N]*/
    int32_t no_start;                       /* skip jump at t0 (src/adjoint_common.jl:761)*/
    int32_t checkpointing;                  /* Backsolve: reset y at checkpoints          */
    int32_t backsolve_ckpt_every_step;      /* 1: checkpoints = all forward steps (sol.t) */
    int32_t mlp_hidden;                     /* FAM_MLP: hidden width (64)                 */
    int32_t cont_cost;                      /* 1: continuous cost g(u) = ca/2 |u|^2 + cb sum(u) is present (accumulate_cost!) */
    double cont_a, cont_b;
    /* preset-time events (DiscreteCallback / PresetTimeCallback with save_positions = (false,false), the hybrid-system
     * adjoint of src/callback_tracking.jl:232-480 for the affine affect family u <- scale .* u + shift; same events for
     * every member; times strictly inside (t0, t1), ascending; adaptive Tsit5 only).  A save time that coincides with
     * an event time records the POST-event state (OrdinaryDiffEq saves after the affect when save_positions is false). */
    int32_t n_events, _pad;
    const double* ev_times;                 /* [E]    */
    const double* ev_scale;                 /* [E][d] */
    const double* ev_shift;                 /* [E][d] */
    const double* ev_pscale;                /* [E][P] or NULL: parameter-changing affect p <- pscale .* p + pshift        */
    const double* ev_pshift;                /* (integrator.p .= 2 .* integrator.p .- 0.5, discrete_callbacks.jl:294-303)  */
    /* per-component coefficients of the named cost family (NULL: the scalars above / zero):
     *   discrete  l(u, p) = sum_j cost_av_j/2 u_j^2 + cost_bv_j u_j + sum_q dgdp_c_q/2 p_q^2 + dgdp_e_q p_q      at every save time
     *   running   g(u, p) = sum_j cont_av_j/2 u_j^2 + cont_bv_j u_j + sum_q cdgdp_c_q/2 p_q^2 + cdgdp_e_q p_q
     * dgdu = a .* u + b, dgdp = c .* p + e  (test/Core7/mixed_costs.jl: g = u1^2 + p1 is a = [2, 0], e = [1, 0, 0, 0]). */
    const double *cost_av, *cost_bv, *cont_av, *cont_bv, *dgdp_c, *dgdp_e, *cdgdp_c, *cdgdp_e;
    /* continuous (root-finding) callback of the named family "coordinate crossing + affine affect" (ContinuousCallback,
     * src/callback_tracking.jl:232-480; docs/src/examples/hybrid_jump/bouncing_ball.md): condition u[cc_idx] - cc_level
     * crossing zero in direction cc_dir (-1 down, +1 up, 0 either); affect u <- cc_scale .* u + cc_shift and, when
     * cc_pcomp >= 0, u[cc_pcomp] <- cc_psign * p[cc_pparam] * u[cc_pcomp] ("v = -e v").  Adaptive Tsit5.  The per-member
     * event times found by the forward solve are returned through cc_found_* (member-local copies of the cfg). */
    int32_t cc_on, cc_idx, cc_dir, cc_pcomp, cc_pparam, cc_found;
    double cc_level, cc_psign;
    const double *cc_scale, *cc_shift;
    /* parameter-dependent condition and additive parameter affect (test/Callbacks2/continuous_callbacks.jl:317-345:
     * condition u[1] - 3/4 p[1], affect u[1] += p[2]): the level is cc_level + cc_lcoef * p[cc_lparam] (cc_lparam < 0: none)
     * and u[cc_acomp] += cc_acoef * p[cc_aparam] (cc_acomp < 0: none) after the affine part */
    int32_t cc_lparam, cc_acomp, cc_aparam, cc_qcomp;
    double cc_lcoef, cc_acoef;
    /* non-linear affect of the reference's tests (test/Callbacks2/continuous_callbacks.jl:222-250, u[2] = u[2]^2):
     * u[cc_qcomp] <- cc_qcoef * u[cc_qcomp]^2 (cc_qcomp < 0: none) instead of the affine map of that component; the
     * reverse pass sees its Jacobian 2 cc_qcoef u-[cc_qcomp] as the event's scale */
    double cc_qcoef;
    /* preset-time events whose affect ADDS A PARAMETER to a state ("Dosing example", test/Callbacks1/discrete_callbacks.jl:401-427:
     * affect(integrator) = integrator.u[1] += integrator.p[2]): after the affine part, u[ev_acomp[e]] += ev_acoef[e] * p[ev_aparam[e]]
     * with the parameters in force before the event (ev_acomp NULL or ev_acomp[e] < 0: none).  Reverse: dG/dp[aparam] += acoef lam+[acomp]. */
    const int32_t *ev_acomp, *ev_aparam;
    const double* ev_acoef;
} oracle_cfg;
#define EV_PADD(c, e, un, pp) do { if ((c)->ev_acomp && (c)->ev_acomp[e] >= 0) (un)[(c)->ev_acomp[e]] += (c)->ev_acoef[e] * (pp)[(c)->ev_aparam[e]]; } while (0)
#define CC_LEVEL(c, p) ((c)->cc_level + ((c)->cc_lparam >= 0 ? (c)->cc_lcoef * (p)[(c)->cc_lparam] : 0.0))
#define COST_A(c, j) ((c)->cost_av ? (c)->cost_av[j] : (c)->cost_a)
#define COST_B(c, j) ((c)->cost_bv ? (c)->cost_bv[j] : (c)->cost_b)
#define CONT_A(c, j) ((c)->cont_av ? (c)->cont_av[j] : (c)->cont_a)
#define CONT_B(c, j) ((c)->cont_bv ? (c)->cont_bv[j] : (c)->cont_b)
/* parameters in force after the first `upto` events */
static void event_params(const oracle_cfg* c, int P, int upto, const double* p0, double* out) {
    for (int q = 0; q < P; q++) out[q] = p0[q];
    if (!c->ev_pscale) return;
    for (int e = 0; e < upto; e++) for (int q = 0; q < P; q++) out[q] = c->ev_pscale[(size_t)e * P + q] * out[q] + c->ev_pshift[(size_t)e * P + q];
}

/* =====================================================================================
 * RHS families: f, hand-differentiated VJPs (what derivative_wrappers.jl's AD back-ends
 * compute; src/derivative_wrappers.jl:256-267), diagonal noise g and its VJPs.
 * ===================================================================================== */
typedef struct { int hidden; } fam_ctx;

static void f_lv(const double* u, const double* p, double t, double* du, const fam_ctx* c) {
    (void)t; (void)c;
    du[0] = p[0] * u[0] - p[1] * u[0] * u[1];
    du[1] = -p[2] * u[1] + p[3] * u[0] * u[1];
}
static void vjp_lv(const double* u, const double* p, double t, const double* l, double* dl, double* dg, const fam_ctx* c) {
    (void)t; (void)c;
    double x = u[0], y = u[1];
    dl[0] = l[0] * (p[0] - p[1] * y) + l[1] * p[3] * y;
    dl[1] = -l[0] * p[1] * x + l[1] * (-p[2] + p[3] * x);
    if (dg) { dg[0] = x * l[0]; dg[1] = -x * y * l[0]; dg[2] = -y * l[1]; dg[3] = x * y * l[1]; }
}
/* bouncing ball (docs/src/examples/hybrid_jump/bouncing_ball.md): x' = v, v' = -p1; p = [gravity, restitution] (the
 * restitution coefficient only enters through the callback's affect) */
static void f_ball(const double* u, const double* p, double t, double* du, const fam_ctx* c) {
    (void)t; (void)c;
    du[0] = u[1]; du[1] = -p[0];
}
static void vjp_ball(const double* u, const double* p, double t, const double* l, double* dl, double* dg, const fam_ctx* c) {
    (void)t; (void)c; (void)u; (void)p;
    dl[0] = 0.0; dl[1] = l[0];
    if (dg) { dg[0] = -l[1]; dg[1] = 0.0; }
}
/* relaxation towards p1 (test/Callbacks2/continuous_callbacks.jl:317-324: f(D,u,p,t) = (D[1] = p[1] - u[1]); p[2] only enters
 * through the callback's affect u[1] += p[2]) */
static void f_relax(const double* u, const double* p, double t, double* du, const fam_ctx* c) {
    (void)t; (void)c;
    du[0] = p[0] - u[0];
}
static void vjp_relax(const double* u, const double* p, double t, const double* l, double* dl, double* dg, const fam_ctx* c) {
    (void)t; (void)c; (void)u; (void)p;
    dl[0] = -l[0];
    if (dg) { dg[0] = l[0]; dg[1] = 0.0; }
}
static void f_lorenz(const double* u, const double* p, double t, double* du, const fam_ctx* c) {
    (void)t; (void)c;
    du[0] = p[0] * (u[1] - u[0]);
    du[1] = u[0] * (p[1] - u[2]) - u[1];
    du[2] = u[0] * u[1] - p[2] * u[2];
}
static void vjp_lorenz(const double* u, const double* p, double t, const double* l, double* dl, double* dg, const fam_ctx* c) {
    (void)t; (void)c;
    dl[0] = -p[0] * l[0] + (p[1] - u[2]) * l[1] + u[1] * l[2];
    dl[1] = p[0] * l[0] - l[1] + u[0] * l[2];
    dl[2] = -u[0] * l[1] - p[2] * l[2];
    if (dg) { dg[0] = (u[1] - u[0]) * l[0]; dg[1] = u[0] * l[1]; dg[2] = -u[2] * l[2]; }
}
static void f_rober(const double* y, const double* k, double t, double* dy, const fam_ctx* c) {
    (void)t; (void)c;
    dy[0] = -k[0] * y[0] + k[2] * y[1] * y[2];
    dy[1] = k[0] * y[0] - k[1] * y[1] * y[1] - k[2] * y[1] * y[2];
    dy[2] = k[1] * y[1] * y[1];
}
static void vjp_rober(const double* y, const double* k, double t, const double* l, double* dl, double* dg, const fam_ctx* c) {
    (void)t; (void)c;
    dl[0] = -k[0] * l[0] + k[0] * l[1];
    dl[1] = k[2] * y[2] * l[0] - (2 * k[1] * y[1] + k[2] * y[2]) * l[1] + 2 * k[1] * y[1] * l[2];
    dl[2] = k[2] * y[1] * l[0] - k[2] * y[1] * l[1];
    if (dg) {
        dg[0] = -y[0] * l[0] + y[0] * l[1];
        dg[1] = -y[1] * y[1] * l[1] + y[1] * y[1] * l[2];
        dg[2] = y[1] * y[2] * l[0] - y[1] * y[2] * l[1];
    }
}
/* Jacobian (row-major J[i*d+j] = df_i/du_j), for Rosenbrock23 */
static void jac_rober(const double* y, const double* k, double* J) {
    J[0] = -k[0];            J[1] = k[2] * y[2];                         J[2] = k[2] * y[1];
    J[3] = k[0];             J[4] = -2 * k[1] * y[1] - k[2] * y[2];      J[5] = -k[2] * y[1];
    J[6] = 0;                J[7] = 2 * k[1] * y[1];                     J[8] = 0;
}
static void jac_lorenz(const double* u, const double* p, double* J) {
    J[0] = -p[0];        J[1] = p[0];  J[2] = 0;
    J[3] = p[1] - u[2];  J[4] = -1;    J[5] = -u[0];
    J[6] = u[1];         J[7] = u[0];  J[8] = -p[2];
}
static void jac_lv(const double* u, const double* p, double* J) {
    J[0] = p[0] - p[1] * u[1];  J[1] = -p[1] * u[0];
    J[2] = p[3] * u[1];         J[3] = -p[2] + p[3] * u[0];
}
/* d/dt of J(y(t)) along ydot:  dJ[i][j] = sum_k d2f_i/du_j du_k * ydot_k  (Hessian contraction) */
static void djac_rober(const double* k, const double* yd, double* dJ) {
    dJ[0] = 0;  dJ[1] = k[2] * yd[2];                        dJ[2] = k[2] * yd[1];
    dJ[3] = 0;  dJ[4] = -2 * k[1] * yd[1] - k[2] * yd[2];    dJ[5] = -k[2] * yd[1];
    dJ[6] = 0;  dJ[7] = 2 * k[1] * yd[1];                    dJ[8] = 0;
}
static void djac_lorenz(const double* yd, double* dJ) {
    dJ[0] = 0;       dJ[1] = 0;      dJ[2] = 0;
    dJ[3] = -yd[2];  dJ[4] = 0;      dJ[5] = -yd[0];
    dJ[6] = yd[1];   dJ[7] = yd[0];  dJ[8] = 0;
}
static void djac_lv(const double* p, const double* yd, double* dJ) {
    dJ[0] = -p[1] * yd[1];  dJ[1] = -p[1] * yd[0];
    dJ[2] = p[3] * yd[1];   dJ[3] = p[3] * yd[0];
}

/* SDE Lotka-Volterra, diagonal noise g_i = p[4+i]*u_i  (test/Core1/concrete_solve_derivatives.jl:737-760) */
static void f_sdelv(const double* u, const double* p, double t, double* du, const fam_ctx* c) { f_lv(u, p, t, du, c); }
static void vjp_sdelv(const double* u, const double* p, double t, const double* l, double* dl, double* dg, const fam_ctx* c) {
    vjp_lv(u, p, t, l, dl, dg, c);
    if (dg) { dg[4] = 0; dg[5] = 0; }
}
static void g_sdelv(const double* u, const double* p, double t, double* g) { (void)t; g[0] = p[4] * u[0]; g[1] = p[5] * u[1]; }
/* Ito->"transformed" drift f - (dg/du)' g  (src/sde_tools.jl:29-66; full correction, no 1/2) */
static void fito_sdelv(const double* u, const double* p, double t, double* du, const fam_ctx* c) {
    f_lv(u, p, t, du, c);
    du[0] -= p[4] * p[4] * u[0];
    du[1] -= p[5] * p[5] * u[1];
}
static void vjpito_sdelv(const double* u, const double* p, double t, const double* l, double* dl, double* dg, const fam_ctx* c) {
    vjp_sdelv(u, p, t, l, dl, dg, c);
    dl[0] -= p[4] * p[4] * l[0];
    dl[1] -= p[5] * p[5] * l[1];
    if (dg) { dg[4] -= 2 * p[4] * u[0] * l[0]; dg[5] -= 2 * p[5] * u[1] * l[1]; }
}
/* diagonal-noise VJP: dlam_i = lam_i dg_i/du_i ; dgradm[P x m] column i = lam_i dg_i/dp
 * (src/derivative_wrappers.jl:1197-1199) */
static void gvjp_sdelv(const double* u, const double* p, double t, const double* l, double* dl, double* dgm /*[m][P]*/) {
    (void)t;
    dl[0] = l[0] * p[4]; dl[1] = l[1] * p[5];
    memset(dgm, 0, sizeof(double) * 12);
    dgm[0 * 6 + 4] = l[0] * u[0];
    dgm[1 * 6 + 5] = l[1] * u[1];
}

/* linear SDE  du_i = p0 u_i dt + p1 u_i dW_i  (test/SDE1/sde_stratonovich.jl:22-31), d = m = any */
static int g_lin_d = 1;
static void f_sdelin(const double* u, const double* p, double t, double* du, const fam_ctx* c) {
    (void)t; for (int i = 0; i < c->hidden; i++) du[i] = p[0] * u[i];
}
static void vjp_sdelin(const double* u, const double* p, double t, const double* l, double* dl, double* dg, const fam_ctx* c) {
    (void)t; double s = 0;
    for (int i = 0; i < c->hidden; i++) { dl[i] = p[0] * l[i]; s += u[i] * l[i]; }
    if (dg) { dg[0] = s; dg[1] = 0; }
}
static void fito_sdelin(const double* u, const double* p, double t, double* du, const fam_ctx* c) {
    (void)t; for (int i = 0; i < c->hidden; i++) du[i] = (p[0] - p[1] * p[1]) * u[i];
}
static void vjpito_sdelin(const double* u, const double* p, double t, const double* l, double* dl, double* dg, const fam_ctx* c) {
    (void)t; double s = 0;
    for (int i = 0; i < c->hidden; i++) { dl[i] = (p[0] - p[1] * p[1]) * l[i]; s += u[i] * l[i]; }
    if (dg) { dg[0] = s; dg[1] = -2 * p[1] * s; }
}

/* MLP  f = W3 tanh(W2 tanh(W1 u + b1) + b2) + b3, column-major weights, p = [W1,b1,W2,b2,W3,b3] */
static void mlp_offsets(int d, int H, int* oW1, int* ob1, int* oW2, int* ob2, int* oW3, int* ob3) {
    *oW1 = 0; *ob1 = H * d; *oW2 = *ob1 + H; *ob2 = *oW2 + H * H; *oW3 = *ob2 + H; *ob3 = *oW3 + d * H;
}
#define MLP_MAXH 256
static void mlp_forward(const double* u, const double* p, int d, int H, double* h1, double* h2, double* out) {
    int oW1, ob1, oW2, ob2, oW3, ob3; mlp_offsets(d, H, &oW1, &ob1, &oW2, &ob2, &oW3, &ob3);
    for (int i = 0; i < H; i++) { double s = p[ob1 + i]; for (int j = 0; j < d; j++) s += p[oW1 + j * H + i] * u[j]; h1[i] = tanh(s); }
    for (int i = 0; i < H; i++) { double s = p[ob2 + i]; for (int j = 0; j < H; j++) s += p[oW2 + j * H + i] * h1[j]; h2[i] = tanh(s); }
    for (int i = 0; i < d; i++) { double s = p[ob3 + i]; for (int j = 0; j < H; j++) s += p[oW3 + j * d + i] * h2[j]; out[i] = s; }
}
static void f_mlp(const double* u, const double* p, double t, double* du, const fam_ctx* c) {
    (void)t; double h1[MLP_MAXH], h2[MLP_MAXH]; mlp_forward(u, p, 2, c->hidden, h1, h2, du);
}
static void vjp_mlp(const double* u, const double* p, double t, const double* l, double* dl, double* dg, const fam_ctx* c) {
    (void)t; const int d = 2, H = c->hidden;
    int oW1, ob1, oW2, ob2, oW3, ob3; mlp_offsets(d, H, &oW1, &ob1, &oW2, &ob2, &oW3, &ob3);
    double h1[MLP_MAXH], h2[MLP_MAXH], out[2], d2[MLP_MAXH], d1[MLP_MAXH];
    mlp_forward(u, p, d, H, h1, h2, out);
    for (int j = 0; j < H; j++) { double s = 0; for (int i = 0; i < d; i++) s += p[oW3 + j * d + i] * l[i]; d2[j] = s * (1 - h2[j] * h2[j]); }
    for (int j = 0; j < H; j++) { double s = 0; for (int i = 0; i < H; i++) s += p[oW2 + j * H + i] * d2[i]; d1[j] = s * (1 - h1[j] * h1[j]); }
    for (int j = 0; j < d; j++) { double s = 0; for (int i = 0; i < H; i++) s += p[oW1 + j * H + i] * d1[i]; dl[j] = s; }
    if (dg) {
        for (int j = 0; j < d; j++) for (int i = 0; i < H; i++) dg[oW1 + j * H + i] = d1[i] * u[j];
        for (int i = 0; i < H; i++) dg[ob1 + i] = d1[i];
        for (int j = 0; j < H; j++) for (int i = 0; i < H; i++) dg[oW2 + j * H + i] = d2[i] * h1[j];
        for (int i = 0; i < H; i++) dg[ob2 + i] = d2[i];
        for (int j = 0; j < H; j++) for (int i = 0; i < d; i++) dg[oW3 + j * d + i] = l[i] * h2[j];
        for (int i = 0; i < d; i++) dg[ob3 + i] = l[i];
    }
}

typedef void (*f_fn)(const double*, const double*, double, double*, const fam_ctx*);
typedef void (*vjp_fn)(const double*, const double*, double, const double*, double*, double*, const fam_ctx*);
typedef struct {
    int d, P, m; fam_ctx ctx; int family;
    f_fn f, f_ito; vjp_fn vjp, vjp_ito;
} family_t;

static int family_init(family_t* F, const oracle_cfg* c) {
    memset(F, 0, sizeof(*F));
    F->family = c->family; F->ctx.hidden = c->mlp_hidden;
    switch (c->family) {
    case FAM_LV:        F->d = 2; F->P = 4; F->f = f_lv; F->vjp = vjp_lv; break;
    case FAM_LORENZ:    F->d = 3; F->P = 3; F->f = f_lorenz; F->vjp = vjp_lorenz; break;
    case FAM_BALL:      F->d = 2; F->P = 2; F->f = f_ball; F->vjp = vjp_ball; break;
    case FAM_RELAX:     F->d = 1; F->P = 2; F->f = f_relax; F->vjp = vjp_relax; break;
    case FAM_ROBERTSON: F->d = 3; F->P = 3; F->f = f_rober; F->vjp = vjp_rober; break;
    case FAM_SDE_LV:    F->d = 2; F->P = 6; F->m = 2; F->f = f_sdelv; F->vjp = vjp_sdelv; F->f_ito = fito_sdelv; F->vjp_ito = vjpito_sdelv; break;
    case FAM_MLP:       F->d = 2; F->P = c->P; F->f = f_mlp; F->vjp = vjp_mlp;
                        if (c->mlp_hidden > MLP_MAXH || c->P != 2 * c->mlp_hidden + c->mlp_hidden + c->mlp_hidden * c->mlp_hidden + c->mlp_hidden + 2 * c->mlp_hidden + 2) return -2;
                        break;
    case FAM_SDE_LINEAR: F->d = c->d; F->P = 2; F->m = c->d; F->ctx.hidden = c->d; F->f = f_sdelin; F->vjp = vjp_sdelin; F->f_ito = fito_sdelin; F->vjp_ito = vjpito_sdelin; break;
    default: return -1;
    }
    if (F->d != c->d || F->P != c->P) return -3;
    (void)g_lin_d;
    return 0;
}
static void fam_g(const family_t* F, const double* u, const double* p, double t, double* g) {
    if (F->family == FAM_SDE_LV) g_sdelv(u, p, t, g);
    else for (int i = 0; i < F->d; i++) g[i] = p[1] * u[i];
}
/* dl_i = lam_i dg_i/du_i ; dgm[i*P + q] = lam_i dg_i/dp_q */
static void fam_gvjp(const family_t* F, const double* u, const double* p, double t, const double* l, double* dl, double* dgm) {
    if (F->family == FAM_SDE_LV) { gvjp_sdelv(u, p, t, l, dl, dgm); return; }
    for (int i = 0; i < F->d; i++) { dl[i] = l[i] * p[1]; dgm[i * 2 + 0] = 0; dgm[i * 2 + 1] = l[i] * u[i]; }
}
static int fam_jac(const family_t* F, const double* u, const double* p, double* J) {
    switch (F->family) {
    case FAM_LV: jac_lv(u, p, J); return 0;
    case FAM_LORENZ: jac_lorenz(u, p, J); return 0;
    case FAM_ROBERTSON: jac_rober(u, p, J); return 0;
    default: return -1;
    }
}
static int fam_djac(const family_t* F, const double* p, const double* yd, double* dJ) {
    switch (F->family) {
    case FAM_LV: djac_lv(p, yd, dJ); return 0;
    case FAM_LORENZ: djac_lorenz(yd, dJ); return 0;
    case FAM_ROBERTSON: djac_rober(p, yd, dJ); return 0;
    default: return -1;
    }
}

/* Parameter Jacobian F[i*P+q] = df_i/dp_q (the `paramjac` of src/derivative_wrappers.jl:284-340) and its derivative along
 * ydot, dF[i*P+q] = sum_k d2f_i/dp_q du_k ydot_k: needed when a Rosenbrock method integrates the AUGMENTED adjoint state
 * (Interpolating / Backsolve), whose Jacobian and time derivative contain F(y(t)). */
static int fam_pjac(const family_t* F, const double* y, double* Fm) {
    switch (F->family) {
    case FAM_LV:      Fm[0] = y[0]; Fm[1] = -y[0] * y[1]; Fm[2] = 0; Fm[3] = 0;   Fm[4] = 0; Fm[5] = 0; Fm[6] = -y[1]; Fm[7] = y[0] * y[1]; return 0;
    case FAM_LORENZ:  Fm[0] = y[1] - y[0]; Fm[1] = 0; Fm[2] = 0;   Fm[3] = 0; Fm[4] = y[0]; Fm[5] = 0;   Fm[6] = 0; Fm[7] = 0; Fm[8] = -y[2]; return 0;
    case FAM_ROBERTSON: Fm[0] = -y[0]; Fm[1] = 0; Fm[2] = y[1] * y[2];   Fm[3] = y[0]; Fm[4] = -y[1] * y[1]; Fm[5] = -y[1] * y[2];   Fm[6] = 0; Fm[7] = y[1] * y[1]; Fm[8] = 0; return 0;
    default: return -1;
    }
}
static int fam_dpjac(const family_t* F, const double* y, const double* yd, double* dF) {
    switch (F->family) {
    case FAM_LV: { double s = yd[0] * y[1] + y[0] * yd[1];
        dF[0] = yd[0]; dF[1] = -s; dF[2] = 0; dF[3] = 0;   dF[4] = 0; dF[5] = 0; dF[6] = -yd[1]; dF[7] = s; return 0; }
    case FAM_LORENZ: dF[0] = yd[1] - yd[0]; dF[1] = 0; dF[2] = 0;   dF[3] = 0; dF[4] = yd[0]; dF[5] = 0;   dF[6] = 0; dF[7] = 0; dF[8] = -yd[2]; return 0;
    case FAM_ROBERTSON: { double s = yd[1] * y[2] + y[1] * yd[2], q = 2 * y[1] * yd[1];
        dF[0] = -yd[0]; dF[1] = 0; dF[2] = s;   dF[3] = yd[0]; dF[4] = -q; dF[5] = -s;   dF[6] = 0; dF[7] = q; dF[8] = 0; return 0; }
    default: return -1;
    }
}

/* =====================================================================================
 * Tsit5 (Tsitouras 2011) tableau and 4th-order dense output  [UPSTREAM OrdinaryDiffEq; SURVEY App. B]
 * ===================================================================================== */
static const double TS_C[7] = {0.0, 0.161, 0.327, 0.9, 0.9800255409045097, 1.0, 1.0};
static const double TS_A[7][6] = {
    {0},
    {0.161},
    {-0.008480655492356989, 0.335480655492357},
    {2.8971530571054935, -6.359448489975075, 4.3622954328695815},
    {5.325864828439257, -11.748883564062828, 7.4955393428898365, -0.09249506636175525},
    {5.86145544294642, -12.92096931784711, 8.159367898576159, -0.071584973281401, -0.028269050394068383},
    {0.09646076681806523, 0.01, 0.4798896504144996, 1.379008574103742, -3.290069515436081, 2.324710524099774}};
/* error estimator weights (b - bhat), including the FSAL stage */
static const double TS_BT[7] = {-0.00178001105222577714, -0.0008164344596567469, 0.007880878010261995,
                                -0.1447110071732629, 0.5823571654525552, -0.45808210592918697, 0.015151515151515152};

void oracle_tsit5_btheta(double th, double* b) {
    double t2 = th * th;
    b[0] = -1.0530884977290216 * th * (th - 1.3299890189751412) * (t2 - 1.4364028541716351 * th + 0.7139816917074209);
    b[1] = 0.1017 * t2 * (t2 - 2.1966568338249754 * th + 1.2949852507374631);
    b[2] = 2.490627285651252793 * t2 * (t2 - 2.38535645472061657 * th + 1.57803468208092486);
    b[3] = -16.54810288924490272 * (th - 1.21712927295533244) * (th - 0.61620406037800089) * t2;
    b[4] = 47.37952196281928122 * (th - 1.203071208372362603) * (th - 0.658047292653547382) * t2;
    b[5] = -34.87065786149660974 * (th - 1.2) * (th - 0.666666666666666667) * t2;
    b[6] = 2.5 * (th - 1.0) * (th - 0.6) * t2;
}
/* derivative of the dense-output weights wrt theta (for ydot(t) of the interpolant) */
static void tsit5_dbtheta(double th, double* db) {
    /* b_i are quartics; differentiate numerically-exactly via expanded coefficients */
    double e = 1e-6, bp[7], bm[7];
    /* quartic => 5-point stencil is exact up to rounding; use Richardson-free central difference of
       a quartic with step e: error O(e^2 * b''') -- instead expand analytically: */
    (void)e; (void)bp; (void)bm;
    /* analytic: b = c * th^a * q(th), handled by product rule on the factored forms */
    double t = th, t2 = th * th;
    {   /* b1 = c t (t - r)(t^2 - s t + w) */
        double c = -1.0530884977290216, r = 1.3299890189751412, s = 1.4364028541716351, w = 0.7139816917074209;
        double A = t, B = t - r, C = t2 - s * t + w;
        db[0] = c * (B * C + A * C + A * B * (2 * t - s));
    }
    {   double c = 0.1017, s = 2.1966568338249754, w = 1.2949852507374631;
        double C = t2 - s * t + w; db[1] = c * (2 * t * C + t2 * (2 * t - s)); }
    {   double c = 2.490627285651252793, s = 2.38535645472061657, w = 1.57803468208092486;
        double C = t2 - s * t + w; db[2] = c * (2 * t * C + t2 * (2 * t - s)); }
    {   double c = -16.54810288924490272, r1 = 1.21712927295533244, r2 = 0.61620406037800089;
        db[3] = c * ((t - r2) * t2 + (t - r1) * t2 + (t - r1) * (t - r2) * 2 * t); }
    {   double c = 47.37952196281928122, r1 = 1.203071208372362603, r2 = 0.658047292653547382;
        db[4] = c * ((t - r2) * t2 + (t - r1) * t2 + (t - r1) * (t - r2) * 2 * t); }
    {   double c = -34.87065786149660974, r1 = 1.2, r2 = 0.666666666666666667;
        db[5] = c * ((t - r2) * t2 + (t - r1) * t2 + (t - r1) * (t - r2) * 2 * t); }
    {   double c = 2.5, r1 = 1.0, r2 = 0.6;
        db[6] = c * ((t - r2) * t2 + (t - r1) * t2 + (t - r1) * (t - r2) * 2 * t); }
}
void oracle_tsit5_tableau(double* c7, double* a7x6, double* bt7) {
    memcpy(c7, TS_C, sizeof(TS_C)); memcpy(a7x6, TS_A, sizeof(TS_A)); memcpy(bt7, TS_BT, sizeof(TS_BT));
}

typedef void (*rhs_fn)(double t, const double* z, double* dz, void* ctx);

/* One Tsit5 step of size h (may be negative) from (t,z).  k is [7][L]; k[0] must hold f(t,z) on
 * entry (FSAL); on exit k[6] = f(t+h, znew). */
static void tsit5_step(rhs_fn rhs, void* ctx, int L, double t, double h, const double* z, double* k, double* znew, double* tmp) {
    for (int s = 1; s < 7; s++) {
        for (int i = 0; i < L; i++) {
            double acc = 0;
            for (int j = 0; j < s; j++) acc += TS_A[s][j] * k[j * L + i];
            tmp[i] = z[i] + h * acc;
        }
        if (s == 6) memcpy(znew, tmp, sizeof(double) * L);
        rhs(t + TS_C[s] * h, tmp, k + s * L, ctx);
    }
}
static void tsit5_dense(int L, double th, double h, const double* z, const double* k, double* out) {
    double b[7]; oracle_tsit5_btheta(th, b);
    for (int i = 0; i < L; i++) {
        double acc = 0;
        for (int j = 0; j < 7; j++) acc += b[j] * k[j * L + i];
        out[i] = z[i] + h * acc;
    }
}
static void tsit5_dense_deriv(int L, double th, const double* k, double* out) {
    double db[7]; tsit5_dbtheta(th, db);
    for (int i = 0; i < L; i++) { double acc = 0; for (int j = 0; j < 7; j++) acc += db[j] * k[j * L + i]; out[i] = acc; }
}

/* =====================================================================================
 * Dense forward solution (what the reference keeps as `sol`, and queries with sol(y,t))
 * ===================================================================================== */
enum { DENSE_TSIT5 = 0, DENSE_ROS23 = 1, DENSE_LINEAR = 2 };
typedef struct {
    int d, n, cap, kind, nk;
    double *t, *u, *k;     /* t[n+1], u[(n+1)*d], k[n*nk*d] */
} dense_t;
static void dense_init(dense_t* S, int d, int kind, int cap) {
    S->d = d; S->n = 0; S->cap = cap; S->kind = kind; S->nk = (kind == DENSE_TSIT5) ? 7 : (kind == DENSE_ROS23 ? 2 : 0);
    S->t = (double*)malloc(sizeof(double) * (cap + 1));
    S->u = (double*)malloc(sizeof(double) * (size_t)(cap + 1) * d);
    S->k = S->nk ? (double*)malloc(sizeof(double) * (size_t)cap * S->nk * d) : NULL;
}
static void dense_grow(dense_t* S) {
    if (S->n < S->cap) return;
    S->cap *= 2;
    S->t = (double*)realloc(S->t, sizeof(double) * (S->cap + 1));
    S->u = (double*)realloc(S->u, sizeof(double) * (size_t)(S->cap + 1) * S->d);
    if (S->nk) S->k = (double*)realloc(S->k, sizeof(double) * (size_t)S->cap * S->nk * S->d);
}
static void dense_free(dense_t* S) { free(S->t); free(S->u); free(S->k); }

static const double ROS_D = 0.29289321881345247559915563789515;  /* 1/(2+sqrt 2) */

/* sol(y, t, continuity = :left | :right)  [UPSTREAM ode_interpolation; SURVEY 8a a6].
 * ts ascending.  right: interval to the right of a knot (theta = 0); left: interval to the left. */
static void dense_eval(const dense_t* S, double t, int right, double* y, double* ydot) {
    int n = S->n, lo = 0, hi = n; /* find i in [0,n-1] */
    int i;
    if (right) { /* last index with ts[idx] <= t, then interval [idx, idx+1] */
        lo = 0; hi = n;  /* invariant ts[lo] <= t (or lo=0) */
        while (hi - lo > 1) { int mid = (lo + hi) / 2; if (S->t[mid] <= t) lo = mid; else hi = mid; }
        i = lo; if (i > n - 1) i = n - 1;
    } else {     /* first index with ts[idx] >= t, interval [idx-1, idx] */
        lo = 0; hi = n;
        while (hi - lo > 1) { int mid = (lo + hi) / 2; if (S->t[mid] >= t) hi = mid; else lo = mid; }
        i = hi - 1; if (i < 0) i = 0;
    }
    double h = S->t[i + 1] - S->t[i];
    double th = (h == 0) ? 1.0 : (t - S->t[i]) / h;
    const double* u = S->u + (size_t)i * S->d;
    if (S->kind == DENSE_TSIT5) {
        const double* k = S->k + (size_t)i * 7 * S->d;
        if (y) tsit5_dense(S->d, th, h, u, k, y);
        if (ydot) tsit5_dense_deriv(S->d, th, k, ydot);
    } else if (S->kind == DENSE_ROS23) {
        const double* k = S->k + (size_t)i * 2 * S->d;
        double c1 = th * (1 - th) / (1 - 2 * ROS_D), c2 = th * (th - 2 * ROS_D) / (1 - 2 * ROS_D);
        double d1 = (1 - 2 * th) / (1 - 2 * ROS_D), d2 = (2 * th - 2 * ROS_D) / (1 - 2 * ROS_D);
        for (int j = 0; j < S->d; j++) {
            if (y) y[j] = u[j] + h * (c1 * k[j] + c2 * k[S->d + j]);
            if (ydot) ydot[j] = d1 * k[j] + d2 * k[S->d + j];
        }
    } else {
        const double* u1 = S->u + (size_t)(i + 1) * S->d;
        for (int j = 0; j < S->d; j++) { if (y) y[j] = u[j] + th * (u1[j] - u[j]); if (ydot) ydot[j] = (u1[j] - u[j]) / h; }
    }
}

/* ---- forward RHS context ---- */
typedef struct { const family_t* F; const double* p; int ito; } fwd_ctx;
static void fwd_rhs(double t, const double* u, double* du, void* c) {
    fwd_ctx* x = (fwd_ctx*)c;
    (x->ito ? x->F->f_ito : x->F->f)(u, x->p, t, du, &x->F->ctx);
}

static double tstop_snap(double tnext, double tstop) {
    double tol = 100 * 2.220446049250313e-16 * fmax(fabs(tnext), fabs(tstop));
    return (fabs(tnext - tstop) <= tol) ? tstop : tnext;
}

/* Fixed-step Tsit5 forward solve, dense (solve(prob, Tsit5(); adaptive=false, dt)).  Grid t0 + n dt,
 * last step shortened to hit t1. */
/* events (evc): preset times ON the dt grid (the caller's responsibility; the reverse solve finds them by time) */
static void forward_tsit5_fixed(const family_t* F, const double* p, const double* u0, double t0, double t1, double dt, dense_t* S, const oracle_cfg* evc) {
    int d = F->d;
    double pcur[64];
    for (int q = 0; q < F->P && q < 64; q++) pcur[q] = p[q];
    const int E = evc ? evc->n_events : 0; int ev = 0;
    fwd_ctx c = {F, (E > 0 && evc->ev_pscale) ? pcur : p, 0};
    int nest = (int)ceil((t1 - t0) / dt) + 2;
    dense_init(S, d, DENSE_TSIT5, nest);
    double* k = (double*)malloc(sizeof(double) * 7 * d), *tmp = (double*)malloc(sizeof(double) * d), *un = (double*)malloc(sizeof(double) * d);
    memcpy(S->u, u0, sizeof(double) * d); S->t[0] = t0;
    fwd_rhs(t0, u0, k, &c);
    double t = t0; int n = 0;
    while (t < t1) {
        double tn = tstop_snap(t0 + (n + 1) * dt, t1);
        if (tn > t1) tn = t1;
        const int at_ev = ev < E && fabs(evc->ev_times[ev] - tn) <= 100 * 2.220446049250313e-16 * fmax(fabs(tn), 1.0);
        if (at_ev) tn = evc->ev_times[ev];       /* the knot IS the event time (the reverse solve stops at exactly this value) */
        double h = tn - t;
        dense_grow(S);
        tsit5_step(fwd_rhs, &c, d, t, h, S->u + (size_t)n * d, k, un, tmp);
        memcpy(S->k + (size_t)n * 7 * d, k, sizeof(double) * 7 * d);
        S->t[n + 1] = tn;
        memcpy(k, k + 6 * d, sizeof(double) * d);  /* FSAL */
        if (at_ev) {
            for (int i = 0; i < d; i++) un[i] = evc->ev_scale[(size_t)ev * d + i] * un[i] + evc->ev_shift[(size_t)ev * d + i];
            EV_PADD(evc, ev, un, c.p);
            ev++;
            if (evc->ev_pscale) event_params(evc, F->P, ev, p, pcur);
            fwd_rhs(tn, un, k, &c);
        }
        memcpy(S->u + (size_t)(n + 1) * d, un, sizeof(double) * d);
        t = tn; n++; S->n = n;
    }
    free(k); free(tmp); free(un);
}

/* Adaptive Tsit5 forward solve (PI controller beta1=7/50, beta2=2/25, gamma=0.9, qmin=1/5, qmax=10;
 * [UPSTREAM OrdinaryDiffEq defaults], error norm = RMS of err/(abstol+reltol*max(|u|,|unew|))). */
/* member-local event list a forward solve with a continuous callback produces */
typedef struct { int n, cap; double *t, *scale, *shift; } cc_events;
static void cc_push(cc_events* E, int d, double tau, const double* sc, const double* sh) {
    if (E->n == E->cap) { E->cap = E->cap ? 2 * E->cap : 16; E->t = (double*)realloc(E->t, sizeof(double) * E->cap);
        E->scale = (double*)realloc(E->scale, sizeof(double) * E->cap * d); E->shift = (double*)realloc(E->shift, sizeof(double) * E->cap * d); }
    E->t[E->n] = tau; memcpy(E->scale + (size_t)E->n * d, sc, sizeof(double) * d); memcpy(E->shift + (size_t)E->n * d, sh, sizeof(double) * d); E->n++;
}
static int forward_tsit5_adaptive_cc(const family_t* F, const double* p, const double* u0, double t0, double t1,
                                     double abstol, double reltol, double dt0, dense_t* S, const oracle_cfg* evc, cc_events* found);
static int forward_tsit5_adaptive(const family_t* F, const double* p, const double* u0, double t0, double t1,
                                  double abstol, double reltol, double dt0, dense_t* S, const oracle_cfg* evc) {
    if (evc && evc->cc_on) return forward_tsit5_adaptive_cc(F, p, u0, t0, t1, abstol, reltol, dt0, S, evc, NULL);
    int d = F->d;
    double pcur[64];                                   /* parameters in force (events may change them) */
    for (int q = 0; q < F->P && q < 64; q++) pcur[q] = p[q];
    fwd_ctx c = {F, (evc && evc->n_events > 0 && evc->ev_pscale) ? pcur : p, 0};
    dense_init(S, d, DENSE_TSIT5, 256);
    double* k = (double*)malloc(sizeof(double) * 7 * d), *tmp = (double*)malloc(sizeof(double) * d), *un = (double*)malloc(sizeof(double) * d);
    memcpy(S->u, u0, sizeof(double) * d); S->t[0] = t0;
    fwd_rhs(t0, u0, k, &c);
    double t = t0, h = dt0 > 0 ? dt0 : 1e-3 * (t1 - t0), qold = 1e-4;
    int n = 0, iters = 0;
    const int E = evc ? evc->n_events : 0; int ev = 0;      /* next event (tstop) ahead of t */
    while (t < t1) {
        if (++iters > 10000000) { free(k); free(tmp); free(un); return -1; }
        int last = 0;
        const double tend = (ev < E) ? evc->ev_times[ev] : t1;      /* event times are tstops of the forward solve */
        if (t + h >= tend || fabs(t + h - tend) < 100 * 2.22e-16 * fabs(tend)) { h = tend - t; last = 1; }
        dense_grow(S);
        const double* u = S->u + (size_t)n * d;
        tsit5_step(fwd_rhs, &c, d, t, h, u, k, un, tmp);
        double e2 = 0;
        for (int i = 0; i < d; i++) {
            double e = 0; for (int j = 0; j < 7; j++) e += TS_BT[j] * k[j * d + i];
            e *= h;
            double sc = abstol + reltol * fmax(fabs(u[i]), fabs(un[i]));
            e2 += (e / sc) * (e / sc);
        }
        double EEst = sqrt(e2 / d);
        double q11 = pow(fmax(EEst, 1e-300), 7.0 / 50.0);
        double q = q11 / pow(qold, 2.0 / 25.0);
        q = fmax(1.0 / 10.0, fmin(1.0 / (1.0 / 5.0), q / 0.9));
        if (EEst <= 1.0) {
            memcpy(S->k + (size_t)n * 7 * d, k, sizeof(double) * 7 * d);     /* k7 = f(u^-) stays with the step that ends at the event */
            t = last ? tend : t + h; S->t[n + 1] = t;
            memcpy(k, k + 6 * d, sizeof(double) * d);
            if (last && ev < E) {
                /* affect!: u <- scale .* u + shift; the next step starts from the post-event state, FSAL re-evaluated */
                for (int i = 0; i < d; i++) un[i] = evc->ev_scale[(size_t)ev * d + i] * un[i] + evc->ev_shift[(size_t)ev * d + i];
                EV_PADD(evc, ev, un, c.p);
                ev++;
                if (evc->ev_pscale) event_params(evc, F->P, ev, p, pcur);
                fwd_rhs(t, un, k, &c);
            }
            memcpy(S->u + (size_t)(n + 1) * d, un, sizeof(double) * d);
            n++; S->n = n;
            qold = fmax(EEst, 1e-4);
            h = h / q;
        } else {
            h = h / fmin(1.0 / (1.0 / 5.0), q11 / 0.9);
        }
    }
    free(k); free(tmp); free(un);
    return 0;
}

/* Adaptive Tsit5 with ONE continuous callback (root-finding on the step's dense output, ContinuousCallback [UPSTREAM
 * OrdinaryDiffEq/DiffEqBase]): after an accepted step [t, t+h] whose end points straddle the condition in the requested
 * direction, the crossing theta* of the interpolant is bisected to the last bit, the step is REDONE with h' = theta* h (so the
 * stored dense data belong to [t, tau]; this is what reeval_internals_due_to_modification! amounts to), the affect is applied
 * to its end state and the post-event state starts the next step (FSAL re-evaluated, controller proposal of the original
 * step kept).  The knot at tau stores the post-event state, k7 = f(u-) stays with the step (as for preset-time events). */
static int forward_tsit5_adaptive_cc(const family_t* F, const double* p, const double* u0, double t0, double t1,
                                     double abstol, double reltol, double dt0, dense_t* S, const oracle_cfg* evc, cc_events* found) {
    int d = F->d;
    fwd_ctx c = {F, p, 0};
    dense_init(S, d, DENSE_TSIT5, 256);
    double* k = (double*)malloc(sizeof(double) * 7 * d), *tmp = (double*)malloc(sizeof(double) * d), *un = (double*)malloc(sizeof(double) * d);
    double sc[8], sh[8], yb[8];
    memcpy(S->u, u0, sizeof(double) * d); S->t[0] = t0;
    fwd_rhs(t0, u0, k, &c);
    double t = t0, h = dt0 > 0 ? dt0 : 1e-3 * (t1 - t0), qold = 1e-4;
    int n = 0, iters = 0, after_event = 0; const int ci = evc->cc_idx;
    const double level = CC_LEVEL(evc, p);
    while (t < t1) {
        if (++iters > 10000000) { free(k); free(tmp); free(un); return -1; }
        int last = 0;
        if (t + h >= t1 || fabs(t + h - t1) < 100 * 2.22e-16 * fabs(t1)) { h = t1 - t; last = 1; }
        dense_grow(S);
        const double* u = S->u + (size_t)n * d;
        tsit5_step(fwd_rhs, &c, d, t, h, u, k, un, tmp);
        double e2 = 0;
        for (int i = 0; i < d; i++) {
            double e = 0; for (int j = 0; j < 7; j++) e += TS_BT[j] * k[j * d + i];
            e *= h;
            double scl = abstol + reltol * fmax(fabs(u[i]), fabs(un[i]));
            e2 += (e / scl) * (e / scl);
        }
        double EEst = sqrt(e2 / d);
        double q11 = pow(fmax(EEst, 1e-300), 7.0 / 50.0);
        double q = q11 / pow(qold, 2.0 / 25.0);
        q = fmax(1.0 / 10.0, fmin(5.0, q / 0.9));
        if (EEst > 1.0) { h = h / fmin(5.0, q11 / 0.9); continue; }
        /* sign changes of the condition on the step's dense output, sampled at theta = j / 10 (interp_points = 10 of
         * ContinuousCallback): a long step may hold a whole flight.  Right after an event the start value is ~0 with a random
         * sign: the first sample decides the side the solution is on. */
        double gprev = u[ci] - level, thprev = 0.0, lo = 0.0, hi = 1.0;
        int hit = 0;
        for (int j = 1; j <= 10 && !hit; j++) {
            const double th = j == 10 ? 1.0 : 0.1 * j;
            double gj;
            if (j == 10) gj = un[ci] - level; else { tsit5_dense(d, th, h, u, k, yb); gj = yb[ci] - level; }
            if (after_event && j == 1) { gprev = gj; thprev = th; continue; }       /* skip the start point */
            if ((evc->cc_dir <= 0 && gprev > 0 && gj <= 0) || (evc->cc_dir >= 0 && gprev < 0 && gj >= 0)) { hit = 1; lo = thprev; hi = th; }
            else { gprev = gj; thprev = th; }
        }
        after_event = 0;
        double tn = last ? t1 : t + h;
        if (hit) {
            const int pos = gprev > 0;                                  /* g(lo) has the sign of gprev */
            for (int it = 0; it < 200; it++) {
                const double mid = 0.5 * (lo + hi);
                if (!(mid > lo && mid < hi)) break;
                tsit5_dense(d, mid, h, u, k, yb);
                const double gm = yb[ci] - level;
                if ((gm > 0) == pos && gm != 0) lo = mid; else hi = mid;
            }
            const double hh = hi * h;                                  /* first representable theta at / past the crossing */
            tsit5_step(fwd_rhs, &c, d, t, hh, u, k, un, tmp);          /* k[0] = f(u) is still valid */
            tn = t + hh;
        }
        memcpy(S->k + (size_t)n * 7 * d, k, sizeof(double) * 7 * d);
        t = tn; S->t[n + 1] = t;
        memcpy(k, k + 6 * d, sizeof(double) * d);
        if (hit) {
            for (int i = 0; i < d; i++) { sc[i] = evc->cc_scale ? evc->cc_scale[i] : 1.0; sh[i] = evc->cc_shift ? evc->cc_shift[i] : 0.0; }
            if (evc->cc_pcomp >= 0) { sc[evc->cc_pcomp] = evc->cc_psign * p[evc->cc_pparam]; sh[evc->cc_pcomp] = 0.0; }
            if (evc->cc_acomp >= 0) sh[evc->cc_acomp] += evc->cc_acoef * p[evc->cc_aparam];
            const double uq = evc->cc_qcomp >= 0 ? un[evc->cc_qcomp] : 0.0;
            for (int i = 0; i < d; i++) un[i] = sc[i] * un[i] + sh[i];
            if (evc->cc_qcomp >= 0) {       /* u_q <- qcoef u_q^2: Jacobian 2 qcoef u_q- is what the reverse pass needs */
                un[evc->cc_qcomp] = evc->cc_qcoef * uq * uq; sc[evc->cc_qcomp] = 2.0 * evc->cc_qcoef * uq; sh[evc->cc_qcomp] = 0.0;
            }
            if (found) cc_push(found, d, t, sc, sh);
            fwd_rhs(t, un, k, &c);
            after_event = 1;
        }
        memcpy(S->u + (size_t)(n + 1) * d, un, sizeof(double) * d);
        n++; S->n = n;
        qold = fmax(EEst, 1e-4);
        h = h / q;
    }
    free(k); free(tmp); free(un);
    return 0;
}

/* ---- small dense LU (partial pivoting) for Rosenbrock W = I - h d J ---- */
static int lu_factor(int n, double* A, int* piv) {
    for (int c = 0; c < n; c++) {
        int pr = c; double mx = fabs(A[c * n + c]);
        for (int r = c + 1; r < n; r++) if (fabs(A[r * n + c]) > mx) { mx = fabs(A[r * n + c]); pr = r; }
        piv[c] = pr;
        if (mx == 0) return -1;
        if (pr != c) for (int j = 0; j < n; j++) { double t = A[c * n + j]; A[c * n + j] = A[pr * n + j]; A[pr * n + j] = t; }
        for (int r = c + 1; r < n; r++) {
            double f = A[r * n + c] / A[c * n + c]; A[r * n + c] = f;
            for (int j = c + 1; j < n; j++) A[r * n + j] -= f * A[c * n + j];
        }
    }
    return 0;
}
static void lu_solve(int n, const double* A, const int* piv, double* b) {
    for (int c = 0; c < n; c++) { int pr = piv[c]; if (pr != c) { double t = b[c]; b[c] = b[pr]; b[pr] = t; } for (int r = c + 1; r < n; r++) b[r] -= A[r * n + c] * b[c]; }
    for (int r = n - 1; r >= 0; r--) { double s = b[r]; for (int j = r + 1; j < n; j++) s -= A[r * n + j] * b[j]; b[r] = s / A[r * n + r]; }
}

/* Generic Rosenbrock23 step (Shampine ode23s form; SURVEY App. B).  jac(t,z,J) row-major L x L,
 * dT = d rhs/dt.  Returns k1,k2 (dense output) and error estimate vector. */
typedef void (*jac_fn)(double t, const double* z, double* J, double* dT, void* ctx);
static int ros23_step(rhs_fn rhs, jac_fn jac, void* ctx, int L, double t, double h, const double* z, const double* f0,
                      double* k1, double* k2, double* znew, double* fnew, double* err, double* work /* L*L + 6L */, int* piv) {
    const double dd = ROS_D, e32 = 6.0 + 1.4142135623730951;
    double* W = work; double* dT = W + L * L; double* f1 = dT + L; double* tmp = f1 + L; double* k3 = tmp + L;
    jac(t, z, W, dT, ctx);
    for (int i = 0; i < L * L; i++) W[i] = -h * dd * W[i];
    for (int i = 0; i < L; i++) W[i * L + i] += 1.0;
    if (lu_factor(L, W, piv)) return -1;
    for (int i = 0; i < L; i++) k1[i] = f0[i] + h * dd * dT[i];
    lu_solve(L, W, piv, k1);
    for (int i = 0; i < L; i++) tmp[i] = z[i] + 0.5 * h * k1[i];
    rhs(t + 0.5 * h, tmp, f1, ctx);
    for (int i = 0; i < L; i++) k2[i] = f1[i] - k1[i];
    lu_solve(L, W, piv, k2);
    for (int i = 0; i < L; i++) { k2[i] += k1[i]; znew[i] = z[i] + h * k2[i]; }
    rhs(t + h, znew, fnew, ctx);
    for (int i = 0; i < L; i++) k3[i] = fnew[i] - e32 * (k2[i] - f1[i]) - 2 * (k1[i] - f0[i]) + h * dd * dT[i];
    lu_solve(L, W, piv, k3);
    for (int i = 0; i < L; i++) err[i] = h / 6.0 * (k1[i] - 2 * k2[i] + k3[i]);
    return 0;
}
static void fwd_jac(double t, const double* u, double* J, double* dT, void* c) {
    fwd_ctx* x = (fwd_ctx*)c; (void)t;
    fam_jac(x->F, u, x->p, J);
    for (int i = 0; i < x->F->d; i++) dT[i] = 0;   /* autonomous families */
}
/* I-controller for Rosenbrock23 (order 2 => exponent 1/3 on the embedded 3rd-order estimate);
 * standard-controller defaults gamma=0.9, qmin=0.2, qmax=10 [UPSTREAM]. */
static double step_factor_I(double EEst, double expo) {
    double q = pow(fmax(EEst, 1e-300), expo) / 0.9;
    return fmax(1.0 / 10.0, fmin(5.0, q));
}
static int forward_ros23(const family_t* F, const double* p, const double* u0, double t0, double t1,
                         double abstol, double reltol, dense_t* S) {
    int d = F->d; fwd_ctx c = {F, p, 0};
    dense_init(S, d, DENSE_ROS23, 256);
    double f0[8], k1[8], k2[8], un[8], fn[8], err[8], work[8 * 8 + 6 * 8]; int piv[8];
    memcpy(S->u, u0, sizeof(double) * d); S->t[0] = t0;
    fwd_rhs(t0, u0, f0, &c);
    double t = t0, h = 1e-6 * (t1 - t0); int n = 0, iters = 0;
    while (t < t1) {
        if (++iters > 10000000) return -1;
        int last = 0;
        if (t + h >= t1 || fabs(t + h - t1) < 100 * 2.22e-16 * fabs(t1)) { h = t1 - t; last = 1; }
        dense_grow(S);
        const double* u = S->u + (size_t)n * d;
        if (ros23_step(fwd_rhs, fwd_jac, &c, d, t, h, u, f0, k1, k2, un, fn, err, work, piv)) return -2;
        double e2 = 0;
        for (int i = 0; i < d; i++) { double sc = abstol + reltol * fmax(fabs(u[i]), fabs(un[i])); e2 += (err[i] / sc) * (err[i] / sc); }
        double EEst = sqrt(e2 / d);
        double q = step_factor_I(EEst, 1.0 / 3.0);
        if (EEst <= 1.0) {
            memcpy(S->k + (size_t)n * 2 * d, k1, sizeof(double) * d);
            memcpy(S->k + (size_t)n * 2 * d + d, k2, sizeof(double) * d);
            memcpy(S->u + (size_t)(n + 1) * d, un, sizeof(double) * d);
            t = last ? t1 : t + h; S->t[n + 1] = t;
            memcpy(f0, fn, sizeof(double) * d);
            n++; S->n = n;
        }
        h = h / q;
    }
    return 0;
}

/* =====================================================================================
 * Adjoint RHS functors (the reference's *SensitivityFunction callables)
 * ===================================================================================== */
typedef struct {
    const family_t* F; const double* p; const dense_t* sol;
    int sensealg; int ito;
    double* y; double* dgtmp;
    long nrhs;
    int cont; double ca[8], cb[8];   /* continuous cost: dlam -= dgdu_continuous(y) = ca .* y + cb (src/derivative_wrappers.jl:1411-1442) */
    double tev;                   /* event time the reverse solve has just crossed: y(tev) is the LEFT limit from here on */
} adj_ctx;

/* z layout: Interp [lam(d); mu(P)], Gauss/Quad [lam(d)], Backsolve [lam(d); mu(P); y(d)] */
static void adj_rhs(double t, const double* z, double* dz, void* c) {
    adj_ctx* x = (adj_ctx*)c; const family_t* F = x->F; int d = F->d, P = F->P;
    vjp_fn vjp = x->ito ? F->vjp_ito : F->vjp;
    x->nrhs++;
    if (x->sensealg == SA_BACKSOLVE) {
        const double* y = z + d + P;                       /* y read from the state (backsolve_adjoint.jl:78-90) */
        vjp(y, x->p, t, z, dz, dz + d, &F->ctx);
        for (int i = 0; i < d + P; i++) dz[i] = -dz[i];      /* :56-57 */
        if (x->cont) for (int i = 0; i < d; i++) dz[i] -= x->ca[i] * y[i] + x->cb[i];
        (x->ito ? F->f_ito : F->f)(y, x->p, t, dz + d + P, &F->ctx);  /* dy = f(y) */
    } else {
        dense_eval(x->sol, t, t != x->tev, x->y, NULL);    /* sol(y,t,continuity=:right); the left limit at an event just crossed */
        if (x->sensealg == SA_INTERPOLATING) {
            vjp(x->y, x->p, t, z, dz, dz + d, &F->ctx);
            for (int i = 0; i < d + P; i++) dz[i] = -dz[i];  /* interpolating_adjoint.jl:166-170 */
        } else {
            vjp(x->y, x->p, t, z, dz, NULL, &F->ctx);        /* gauss_adjoint.jl:123, quadrature_adjoint.jl:41 */
            for (int i = 0; i < d; i++) dz[i] = -dz[i];
        }
        if (x->cont) for (int i = 0; i < d; i++) dz[i] -= x->ca[i] * x->y[i] + x->cb[i];   /* accumulate_cost!: dlam -= g_u */
    }
}
/* Jacobian and time derivative of adj_rhs for Rosenbrock23 on the adjoint ODE (Gauss/Quad state = lam):
 * d/dlam = -J(y(t))^T (src/quadrature_adjoint.jl:170-192), d/dt = -(dJ/dt)^T lam with ydot from the
 * forward interpolant (what ForwardDiff-through-sol(t) yields, src/quadrature_adjoint.jl:67-71). */
static void adj_jac(double t, const double* z, double* Jout, double* dT, void* c) {
    adj_ctx* x = (adj_ctx*)c; const family_t* F = x->F; const int d = F->d, P = F->P;
    double y[8], yd[8], J[64], dJ[64], Fm[64], dF[64];
    if (x->sensealg == SA_BACKSOLVE) {
        /* z = [lam; mu; y], autonomous: dT = 0.  Rows: lam' = -J(y)'lam (- ca y - cb), mu' = -F(y)'lam, y' = f(y). */
        const int L = 2 * d + P; const double* yy = z + d + P;
        for (int i = 0; i < L * L; i++) Jout[i] = 0;
        for (int i = 0; i < L; i++) dT[i] = 0;
        fam_jac(F, yy, x->p, J); fam_pjac(F, yy, Fm);
        for (int i = 0; i < d; i++) for (int j = 0; j < d; j++) { Jout[i * L + j] = -J[j * d + i]; Jout[(d + P + i) * L + (d + P + j)] = J[i * d + j]; }
        for (int q = 0; q < P; q++) for (int j = 0; j < d; j++) Jout[(d + q) * L + j] = -Fm[j * P + q];
        for (int j = 0; j < d; j++) {               /* column of d/dy_j: Hessian contractions with lam */
            double e[8] = {0}; e[j] = 1.0;
            fam_djac(F, x->p, e, dJ); fam_dpjac(F, yy, e, dF);
            for (int i = 0; i < d; i++) { double a = 0; for (int k = 0; k < d; k++) a -= dJ[k * d + i] * z[k]; Jout[i * L + (d + P + j)] = a - (x->cont && i == j ? x->ca[i] : 0.0); }
            for (int q = 0; q < P; q++) { double a = 0; for (int k = 0; k < d; k++) a -= dF[k * P + q] * z[k]; Jout[(d + q) * L + (d + P + j)] = a; }
        }
        return;
    }
    dense_eval(x->sol, t, t != x->tev, y, yd);
    fam_jac(F, y, x->p, J); fam_djac(F, x->p, yd, dJ);
    const int L = (x->sensealg == SA_INTERPOLATING) ? d + P : d;
    if (L > d) for (int i = 0; i < L * L; i++) Jout[i] = 0;
    for (int i = 0; i < d; i++) {
        double s = 0;
        for (int j = 0; j < d; j++) { Jout[i * L + j] = -J[j * d + i]; s -= dJ[j * d + i] * z[j]; }
        dT[i] = s - (x->cont ? x->ca[i] * yd[i] : 0.0);          /* d/dt of -(ca y(t) + cb) */
    }
    if (L > d) {                                   /* InterpolatingAdjoint: mu' = -F(y(t))' lam */
        fam_pjac(F, y, Fm); fam_dpjac(F, y, yd, dF);
        for (int q = 0; q < P; q++) {
            double s = 0;
            for (int j = 0; j < d; j++) { Jout[(d + q) * L + j] = -Fm[j * P + q]; s -= dF[j * P + q] * z[j]; }
            dT[d + q] = s;
        }
    }
}

/* cotangent at save index k for one trajectory (dgdu_discrete; src/concrete_solve.jl:778-947 or user dg) */
static void cost_grad(const oracle_cfg* c, const double* dLdu_k /* [d] gathered or NULL */, const double* y, double* out) {
    if (c->cost_kind == COST_EXPLICIT) for (int i = 0; i < c->d; i++) out[i] = dLdu_k[i];
    else for (int i = 0; i < c->d; i++) out[i] = COST_A(c, i) * y[i] + COST_B(c, i);
}

/* ---- adjoint dense record (QuadratureAdjoint keeps adj_sol with save_everystep) ---- */
typedef struct { int n, cap, L, nk; double *t0, *h, *z, *k; int kind; } adjdense_t;
static void adjdense_init(adjdense_t* A, int L, int kind) {
    A->n = 0; A->cap = 256; A->L = L; A->kind = kind; A->nk = kind == DENSE_TSIT5 ? 7 : 2;
    A->t0 = (double*)malloc(sizeof(double) * A->cap); A->h = (double*)malloc(sizeof(double) * A->cap);
    A->z = (double*)malloc(sizeof(double) * A->cap * L); A->k = (double*)malloc(sizeof(double) * (size_t)A->cap * A->nk * L);
}
static void adjdense_push(adjdense_t* A, double t0, double h, const double* z, const double* k) {
    if (A->n == A->cap) {
        A->cap *= 2;
        A->t0 = (double*)realloc(A->t0, sizeof(double) * A->cap); A->h = (double*)realloc(A->h, sizeof(double) * A->cap);
        A->z = (double*)realloc(A->z, sizeof(double) * A->cap * A->L); A->k = (double*)realloc(A->k, sizeof(double) * (size_t)A->cap * A->nk * A->L);
    }
    A->t0[A->n] = t0; A->h[A->n] = h;
    memcpy(A->z + (size_t)A->n * A->L, z, sizeof(double) * A->L);
    memcpy(A->k + (size_t)A->n * A->nk * A->L, k, sizeof(double) * A->nk * A->L);
    A->n++;
}
static void adjdense_free(adjdense_t* A) { free(A->t0); free(A->h); free(A->z); free(A->k); }
/* adj_sol(lam, t): steps are stored in descending time; step i spans [t0_i + h_i, t0_i] (h_i < 0) */
static void adjdense_eval(const adjdense_t* A, double t, double* lam) {
    int lo = 0, hi = A->n - 1;
    while (lo < hi) { int mid = (lo + hi) / 2; if (A->t0[mid] + A->h[mid] <= t) hi = mid; else lo = mid + 1; }
    int i = lo; double th = (t - A->t0[i]) / A->h[i];
    const double* z = A->z + (size_t)i * A->L; const double* k = A->k + (size_t)i * A->nk * A->L;
    if (A->kind == DENSE_TSIT5) tsit5_dense(A->L, th, A->h[i], z, k, lam);
    else {
        double c1 = th * (1 - th) / (1 - 2 * ROS_D), c2 = th * (th - 2 * ROS_D) / (1 - 2 * ROS_D);
        for (int j = 0; j < A->L; j++) lam[j] = z[j] + A->h[i] * (c1 * k[j] + c2 * k[A->L + j]);
    }
}

/* ---- QuadGK: adaptive Gauss-Kronrod (7,15), vector valued, 2-norm error [UPSTREAM QuadGK] ---- */
static const double XGK[8] = {0.991455371120812639206854697526329, 0.949107912342758524526189684047851,
    0.864864423359769072789712788640926, 0.741531185599394439863864773280788, 0.586087235467691130294144838258730,
    0.405845151377397166906606412076961, 0.207784955007898467600689403773245, 0.0};
static const double WGK[8] = {0.022935322010529224963732008058970, 0.063092092629978553290700663189204,
    0.104790010322250183839876322541518, 0.140653259715525918745189590510238, 0.169004726639267902826583426598550,
    0.190350578064785409913256402421014, 0.204432940075298892414161999234649, 0.209482141084727828012999174891714};
static const double WG[4] = {0.129484966168869693270611432679082, 0.279705391489276667901467771423780,
    0.381830050505118944950369775488975, 0.417959183673469387755102040816327};
typedef void (*integrand_fn)(double t, double* out, void* ctx);
typedef struct { double a, b, err; double* I; } gkseg;
static void gk15(integrand_fn f, void* ctx, int P, double a, double b, double* Ik, double* err, double* w1, double* w2, double* Ig) {
    double c = 0.5 * (a + b), hl = 0.5 * (b - a);
    for (int q = 0; q < P; q++) { Ik[q] = 0; Ig[q] = 0; }
    f(c, w1, ctx);
    for (int q = 0; q < P; q++) { Ik[q] += WGK[7] * w1[q]; Ig[q] += WG[3] * w1[q]; }
    for (int j = 0; j < 7; j++) {
        f(c - hl * XGK[j], w1, ctx); f(c + hl * XGK[j], w2, ctx);
        for (int q = 0; q < P; q++) {
            Ik[q] += WGK[j] * (w1[q] + w2[q]);
            if (j & 1) Ig[q] += WG[j / 2] * (w1[q] + w2[q]);
        }
    }
    double e2 = 0;
    for (int q = 0; q < P; q++) { Ik[q] *= hl; Ig[q] *= hl; e2 += (Ik[q] - Ig[q]) * (Ik[q] - Ig[q]); }
    *err = sqrt(e2);
}
/* QuadGK.jl's adapt loop: pop the largest-error segment, bisect, and update the running totals INCREMENTALLY
 * (I = (I - s.I) + s1.I + s2.I, E likewise); the running I is what is returned. */
/* diagnostics: integrand evaluations spent by all quadgk calls since the last reset (sizing of the device kernel) */
static long g_quadgk_evals = 0;
long oracle_quadgk_evals(int reset) { long v = g_quadgk_evals; if (reset) g_quadgk_evals = 0; return v; }
long oracle_quadgk(integrand_fn f, void* ctx, int P, double a, double b, double atol, double rtol, double* out) {
    int cap = 64, n = 1; long evals = 15;
    gkseg* S = (gkseg*)malloc(sizeof(gkseg) * cap);
    double* w1 = (double*)malloc(sizeof(double) * P * 5), *w2 = w1 + P, *Ig = w2 + P, *Il = Ig + P, *Ir = Il + P;
    S[0].a = a; S[0].b = b; S[0].I = (double*)malloc(sizeof(double) * P);
    gk15(f, ctx, P, a, b, S[0].I, &S[0].err, w1, w2, Ig);
    double E = S[0].err;
    for (int q = 0; q < P; q++) out[q] = S[0].I[q];
    for (;;) {
        double nI = 0;
        for (int q = 0; q < P; q++) nI += out[q] * out[q];
        nI = sqrt(nI);
        if (E <= fmax(atol, rtol * nI) || evals > 10000000 || n > 1000000) break;
        int w = 0; for (int i = 1; i < n; i++) if (S[i].err > S[w].err) w = i;
        double mid = 0.5 * (S[w].a + S[w].b);
        if (!(mid > fmin(S[w].a, S[w].b) && mid < fmax(S[w].a, S[w].b))) break;
        if (n + 1 > cap) { cap *= 2; S = (gkseg*)realloc(S, sizeof(gkseg) * cap); }
        double el, er;
        gk15(f, ctx, P, S[w].a, mid, Il, &el, w1, w2, Ig);
        gk15(f, ctx, P, mid, S[w].b, Ir, &er, w1, w2, Ig);
        E += (el + er) - S[w].err;
        S[n].I = (double*)malloc(sizeof(double) * P);
        for (int q = 0; q < P; q++) { out[q] += (Il[q] + Ir[q]) - S[w].I[q]; S[w].I[q] = Il[q]; S[n].I[q] = Ir[q]; }
        S[n].a = mid; S[n].b = S[w].b; S[n].err = er;
        S[w].b = mid; S[w].err = el;
        n++; evals += 30;
    }
    for (int i = 0; i < n; i++) free(S[i].I);
    free(S); free(w1);
#pragma omp atomic
    g_quadgk_evals += evals;
    return evals;
}
typedef struct { const family_t* F; const double* p; const dense_t* sol; const adjdense_t* adj; double* y; double* lam; double* dl; } quad_ctx;
/* AdjointSensitivityIntegrand (src/quadrature_adjoint.jl:486-502): out = (df/dp)(y(t))' lam(t) */
static void quad_integrand(double t, double* out, void* c) {
    quad_ctx* x = (quad_ctx*)c;
    dense_eval(x->sol, t, 0, x->y, NULL);
    adjdense_eval(x->adj, t, x->lam);
    x->F->vjp(x->y, x->p, t, x->lam, x->dl, out, &x->F->ctx);
}

/* Gauss-Legendre rules used by IntegratingSumCallback: n = (alg_order+1) div 2 [UPSTREAM DiffEqCallbacks] */
static const double GL1_X[1] = {0.0}, GL1_W[1] = {2.0};
static const double GL3_X[3] = {-0.7745966692414834, 0.0, 0.7745966692414834};
static const double GL3_W[3] = {0.5555555555555556, 0.8888888888888888, 0.5555555555555556};

/* =====================================================================================
 * ODE adjoint driver for ONE ensemble member:  _adjoint_sensitivities
 *   (src/sensitivity_interface.jl:426-526, src/gauss_adjoint.jl:766-870, src/quadrature_adjoint.jl:510-633)
 * ts[K] ascending save times; dL[K*d] cotangents for this member (or NULL for COST_AFFINE)
 * ===================================================================================== */
/* ---- GaussKronrodAdjoint: IntegratingGKSumCallback [UPSTREAM DiffEqCallbacks >= 4.18, not vendored; restated from its
 * published source].  After every accepted step of the reverse solve the integrand is integrated over [tprev, t] with a
 * Gauss-Kronrod pair of n = div(alg_order + 1, 2) Gauss points (Tsit5: G3/K7, Rosenbrock23: G1/K3) evaluated with the
 * integrator's own interpolant; if sum(abs(K - G)) >= tol (1e-7, the callback's default) the interval is bisected and
 * both halves are integrated recursively, otherwise K is added to the running sum (gauss_adjoint.jl:820-825). ---- */
static const double GK7_X[7] = {-0.960491268708020283423507092629080, -0.774596669241483377035853079956480, -0.405845151377397166906606412076961, 0.0,
                                0.405845151377397166906606412076961, 0.774596669241483377035853079956480, 0.960491268708020283423507092629080};
static const double GK7_W[7] = {0.104656226026467265193823857192073, 0.268488089868333440728569280666710, 0.401397414775962222905051818618432,
                                0.450916538658474142345110087045571, 0.401397414775962222905051818618432, 0.268488089868333440728569280666710,
                                0.104656226026467265193823857192073};
static const double GK7_G[3] = {0.555555555555555555555555555555556, 0.888888888888888888888888888888889, 0.555555555555555555555555555555556};
static const double GK3_X[3] = {-0.774596669241483377035853079956480, 0.0, 0.774596669241483377035853079956480};
static const double GK3_W[3] = {0.555555555555555555555555555555556, 0.888888888888888888888888888888889, 0.555555555555555555555555555555556};
static const double GK3_G[1] = {2.0};
#define GK_TOL 1e-7
typedef void (*gk_node_fn)(double tj, double* out /*[P]*/, void* ctx);
static void integrate_gk(gk_node_fn f, void* ctx, int P, int order, double bl, double br, double* accum, int depth) {
    const int np = 2 * order + 1;
    const double* X = order == 3 ? GK7_X : GK3_X; const double* W = order == 3 ? GK7_W : GK3_W; const double* G = order == 3 ? GK7_G : GK3_G;
    double K[64], Gs[64], v[64];
    for (int q = 0; q < P; q++) { K[q] = 0; Gs[q] = 0; }
    for (int i = 0; i < np; i++) {
        double tj = 0.5 * (br - bl) * X[i] + 0.5 * (bl + br);
        f(tj, v, ctx);
        for (int q = 0; q < P; q++) K[q] += W[i] * v[q];
        if (i % 2 == 1) for (int q = 0; q < P; q++) Gs[q] += G[i / 2] * v[q];      /* every second Kronrod point is a Gauss point */
    }
    double err = 0;
    for (int q = 0; q < P; q++) { K[q] *= 0.5 * (br - bl); Gs[q] *= 0.5 * (br - bl); err += fabs(K[q] - Gs[q]); }
    if (err < GK_TOL || depth >= 30) { for (int q = 0; q < P; q++) accum[q] += K[q]; return; }
    const double mid = 0.5 * (bl + br);
    integrate_gk(f, ctx, P, order, bl, mid, accum, depth + 1);
    integrate_gk(f, ctx, P, order, mid, br, accum, depth + 1);
}
typedef struct { const family_t* F; const double* p; const dense_t* sol; int ros, d, L; double t, hs; const double* z; const double* k; double* y; double* lamq; double* dlq; } gkstep_ctx;
static void gkstep_node(double tj, double* out, void* c) {
    gkstep_ctx* x = (gkstep_ctx*)c; const int d = x->d;
    const double th = (tj - x->t) / x->hs;
    if (!x->ros) tsit5_dense(d, th, x->hs, x->z, x->k, x->lamq);
    else { const double c1 = th * (1 - th) / (1 - 2 * 0.29289321881345247559915563789515), c2 = th * (th - 2 * 0.29289321881345247559915563789515) / (1 - 2 * 0.29289321881345247559915563789515);
           for (int i = 0; i < d; i++) x->lamq[i] = x->z[i] + x->hs * (c1 * x->k[i] + c2 * x->k[x->L + i]); }
    dense_eval(x->sol, tj, 0, x->y, NULL);
    x->F->vjp(x->y, x->p, tj, x->lamq, x->dlq, out, &x->F->ctx);
    for (int q = 0; q < x->F->P; q++) out[q] = -out[q];                            /* GaussIntegrand: out = -F'lam */
}

static int adjoint_ode_member(const oracle_cfg* cfg, const family_t* F, const double* p_in, const dense_t* sol,
                              const double* ts, const double* dL, double* du0, double* dp, long* nrhs_out) {
    const int d = F->d, P = F->P, K = cfg->K, sa = cfg->sensealg;
    /* parameters in force on the segment the reverse solve is in: after all events at t = T, re-derived from the caller's p
     * at every event crossed (the reference's reset_p, src/interpolating_adjoint.jl:748-823) */
    double pcur_small[64]; double* pcur = pcur_small; int p_events = (cfg->n_events > 0 && cfg->ev_pscale != NULL);
    if (p_events && P > 64) return -13;
    if (p_events) event_params(cfg, P, cfg->n_events, p_in, pcur);
    const double* p = p_events ? pcur : p_in;
    const int L = (sa == SA_INTERPOLATING) ? d + P : (sa == SA_BACKSOLVE ? 2 * d + P : d);
    const int ros = (cfg->stepper == ST_ROSENBROCK23);
    const int adaptive = (cfg->stepper == ST_TSIT5_ADAPTIVE) || ros;
    if (ros && F->family != FAM_LV && F->family != FAM_LORENZ && F->family != FAM_ROBERTSON) return -10;   /* analytic Jacobians of the adjoint system */
    double T = cfg->t1, t0 = cfg->t0;
    double* z = (double*)calloc(L, sizeof(double)), *zn = (double*)malloc(sizeof(double) * L), *tmp = (double*)malloc(sizeof(double) * L);
    double* k = (double*)malloc(sizeof(double) * 7 * L);
    double* ybuf = (double*)malloc(sizeof(double) * (d + 2 * P + 4 * d + 8));
    double* gu = ybuf + d, *lamq = gu + d, *dlq = lamq + d, *integ = dlq + d, *acc = integ + P;
    adj_ctx ctx = {F, p, sol, sa, 0, ybuf, NULL, 0, cfg->cont_cost, {0}, {0}, INFINITY};
    for (int j = 0; j < d && j < 8; j++) { ctx.ca[j] = CONT_A(cfg, j); ctx.cb[j] = CONT_B(cfg, j); }
    int evc = cfg->n_events - 1;     /* next event below t */
    if (cfg->n_events > 0 && ((cfg->stepper != ST_TSIT5_ADAPTIVE && cfg->stepper != ST_TSIT5_FIXED) || sa == SA_QUADRATURE)) return -11;
    if (cfg->cc_on && (cfg->stepper != ST_TSIT5_ADAPTIVE || sa == SA_QUADRATURE)) return -12;
    for (int q = 0; q < P; q++) acc[q] = 0;
    adjdense_t adj; int have_adj = (sa == SA_QUADRATURE);
    if (have_adj) adjdense_init(&adj, L, ros ? DENSE_ROS23 : DENSE_TSIT5);

    if (sa == SA_BACKSOLVE) memcpy(z + d + P, sol->u + (size_t)sol->n * d, sizeof(double) * d);   /* y(T) = sol.u[end] (backsolve_adjoint.jl:229-231) */

    int cur = K - 1;    /* cur_time (adjoint_common.jl:841) */
    /* checkpoint cursor for Backsolve: the forward knots (sol.t) or the save times */
    int ck = sol->n;
    double t = T;
    /* PresetTimeCallback fires at initialisation when the start time is a preset time */
#define APPLY_JUMP_IF_AT(tt)                                                                               \
    while (cur >= 0 && fabs(ts[cur] - (tt)) <= 100 * 2.220446049250313e-16 * fmax(fabs(tt), 1.0)) {       \
        if (!(cfg->no_start && cur == 0 && sa != SA_BACKSOLVE)) {                                          \
            const double* yy;                                                                              \
            if (sa == SA_BACKSOLVE) yy = z + d + P; else { dense_eval(sol, ts[cur], 1, ybuf, NULL); yy = ybuf; } \
            cost_grad(cfg, dL ? dL + (size_t)cur * d : NULL, yy, gu);                                      \
            for (int i = 0; i < d; i++) z[i] += gu[i];                                                     \
        }                                                                                                  \
        cur--; fsal_ok = 0;                                                                                \
    }
#define APPLY_CKPT_IF_AT(tt)                                                                               \
    if (sa == SA_BACKSOLVE && cfg->checkpointing) {                                                        \
        if (cfg->backsolve_ckpt_every_step) {                                                              \
            while (ck >= 0 && sol->t[ck] > (tt) + 100 * 2.220446049250313e-16 * fmax(fabs(tt), 1.0)) ck--; \
            if (ck >= 0 && fabs(sol->t[ck] - (tt)) <= 100 * 2.220446049250313e-16 * fmax(fabs(tt), 1.0)) { \
                memcpy(z + d + P, sol->u + (size_t)ck * d, sizeof(double) * d); fsal_ok = 0; }             \
        } else if (cur >= 0 && fabs(ts[cur] - (tt)) <= 100 * 2.220446049250313e-16 * fmax(fabs(tt), 1.0)) { \
            dense_eval(sol, ts[cur], (evc >= 0 && cfg->ev_times[evc] == ts[cur]), z + d + P, NULL); fsal_ok = 0; /* post-event state at a coinciding event */ \
        }                                                                                                  \
    }
    /* reverse affect of a preset-time event (callback_tracking.jl:232-480 for u <- s .* u + c): lam(tau-) = s .* lam(tau+);
     * Backsolve takes y(tau-) from the forward solution (the reference stores it as `uleft` in the TrackedAffect).
     * Runs after the checkpoint reset and the loss jump of the same time (the saved state at tau is post-event). */
#define APPLY_EVENT_IF_AT(tt)                                                                              \
    while (evc >= 0 && fabs(cfg->ev_times[evc] - (tt)) <= 100 * 2.220446049250313e-16 * fmax(fabs(tt), 1.0)) { \
        if (cfg->cc_on) {                                                                                  \
            /* state-dependent event time (src/callback_tracking.jl:232-480, the implicit correction): with u+ = a(u-, p),   \
             * g(u-) = 0:  lam- = A'lam+ - dg' [(A f- - f+)' lam+] / (dg . f-),  dG/dp += (da/dp)' lam+ */                  \
            double um[8], up[8], fm[8], fp_[8]; double wl = 0;                                             \
            dense_eval(sol, cfg->ev_times[evc], 0, um, NULL); dense_eval(sol, cfg->ev_times[evc], 1, up, NULL); \
            F->f(um, p, (tt), fm, &F->ctx); F->f(up, p, (tt), fp_, &F->ctx);                               \
            for (int i = 0; i < d; i++) wl += (cfg->ev_scale[(size_t)evc * d + i] * fm[i] - fp_[i]) * z[i]; \
            if (cfg->cc_pcomp >= 0) {                                                                      \
                const double gpar = cfg->cc_psign * um[cfg->cc_pcomp] * z[cfg->cc_pcomp];                  \
                if (sa == SA_INTERPOLATING || sa == SA_BACKSOLVE) z[d + cfg->cc_pparam] += gpar; else acc[cfg->cc_pparam] += gpar; \
            }                                                                                              \
            if (cfg->cc_acomp >= 0) {    /* u+[acomp] += acoef p[aparam]: (da/dp)' lam+ */                    \
                const double gadd = cfg->cc_acoef * z[cfg->cc_acomp];                                      \
                if (sa == SA_INTERPOLATING || sa == SA_BACKSOLVE) z[d + cfg->cc_aparam] += gadd; else acc[cfg->cc_aparam] += gadd; \
            }                                                                                              \
            if (cfg->cc_lparam >= 0) {   /* g = u_i - level - lcoef p[lparam]: -(dg/dp) w / (dg/du . f-) */   \
                const double glev = cfg->cc_lcoef * wl / fm[cfg->cc_idx];                                  \
                if (sa == SA_INTERPOLATING || sa == SA_BACKSOLVE) z[d + cfg->cc_lparam] += glev; else acc[cfg->cc_lparam] += glev; \
            }                                                                                              \
            for (int i = 0; i < d; i++) z[i] *= cfg->ev_scale[(size_t)evc * d + i];                        \
            z[cfg->cc_idx] -= wl / fm[cfg->cc_idx];                                                        \
            if (sa == SA_BACKSOLVE) memcpy(z + d + P, um, sizeof(double) * d);                             \
            ctx.tev = (tt); evc--; fsal_ok = 0; continue;                                                  \
        }                                                                                                  \
        const double ev_gadd = (cfg->ev_acomp && cfg->ev_acomp[evc] >= 0) ? cfg->ev_acoef[evc] * z[cfg->ev_acomp[evc]] : 0.0; /* (da/dp)'lam+ */ \
        for (int i = 0; i < d; i++) z[i] *= cfg->ev_scale[(size_t)evc * d + i];                            \
        if (sa == SA_BACKSOLVE) dense_eval(sol, cfg->ev_times[evc], 0, z + d + P, NULL);                   \
        if (p_events) {   /* p+ = s_p .* p- + c_p: dG/dp- = s_p .* dG/dp+ (+ what accumulates below tau with p-) */ \
            for (int q = 0; q < P; q++) {                                                                  \
                if (sa == SA_INTERPOLATING || sa == SA_BACKSOLVE) z[d + q] *= cfg->ev_pscale[(size_t)evc * P + q]; \
                else acc[q] *= cfg->ev_pscale[(size_t)evc * P + q];                                        \
            }                                                                                              \
            event_params(cfg, P, evc, p_in, pcur);                                                         \
        }                                                                                                  \
        if (cfg->ev_acomp && cfg->ev_acomp[evc] >= 0) {    /* wrt the parameters in force before the event */ \
            if (sa == SA_INTERPOLATING || sa == SA_BACKSOLVE) z[d + cfg->ev_aparam[evc]] += ev_gadd; else acc[cfg->ev_aparam[evc]] += ev_gadd; \
        }                                                                                                  \
        ctx.tev = (tt); evc--; fsal_ok = 0;                                                                \
    }
    int fsal_ok = 0;
    APPLY_CKPT_IF_AT(t);
    APPLY_JUMP_IF_AT(t);

    double h = -fabs(cfg->dt);
    if (adaptive && cfg->dt <= 0) h = -1e-4 * (T - t0);
    double qold = 1e-4; long iters = 0; int rc = 0;
    double f0[16], k1r[16], k2r[16], fnr[16], errv[16], work[16 * 16 + 6 * 16]; int piv[16];
    while (t > t0) {
        if (++iters > 50000000) { rc = -20; break; }
        /* next tstop: next save time below t (PresetTimeCallback tstops), else t0.  For Backsolve with
           per-step checkpoints every forward knot is a tstop as well. */
        double tstop = t0;
        if (cur >= 0 && ts[cur] < t && ts[cur] > tstop) tstop = ts[cur];
        if (evc >= 0 && cfg->ev_times[evc] < t && cfg->ev_times[evc] > tstop) tstop = cfg->ev_times[evc];
        if (sa == SA_BACKSOLVE && cfg->checkpointing && cfg->backsolve_ckpt_every_step) {
            int c2 = ck; while (c2 >= 0 && sol->t[c2] >= t - 100 * 2.220446049250313e-16 * fmax(fabs(t), 1.0)) c2--;
            if (c2 >= 0 && sol->t[c2] > tstop) tstop = sol->t[c2];
        }
        double tn = tstop_snap(t + h, tstop);
        if (tn < tstop) tn = tstop;
        double hs = tn - t;
        if (!ros) {
            if (!fsal_ok) adj_rhs(t, z, k, &ctx);
            tsit5_step(adj_rhs, &ctx, L, t, hs, z, k, zn, tmp);
            if (adaptive) {
                double e2 = 0;
                for (int i = 0; i < L; i++) {
                    double e = 0; for (int j = 0; j < 7; j++) e += TS_BT[j] * k[j * L + i];
                    e *= hs; double sc = cfg->abstol + cfg->reltol * fmax(fabs(z[i]), fabs(zn[i]));
                    e2 += (e / sc) * (e / sc);
                }
                double EEst = sqrt(e2 / L);
                double q11 = pow(fmax(EEst, 1e-300), 7.0 / 50.0);
                double q = fmax(0.1, fmin(5.0, q11 / pow(qold, 2.0 / 25.0) / 0.9));
                if (EEst > 1.0) { h = hs / fmin(5.0, q11 / 0.9); fsal_ok = 1; continue; }
                qold = fmax(EEst, 1e-4); h = hs / q;
            }
        } else {
            if (!fsal_ok) adj_rhs(t, z, f0, &ctx);
            if (ros23_step(adj_rhs, adj_jac, &ctx, L, t, hs, z, f0, k1r, k2r, zn, fnr, errv, work, piv)) { rc = -21; break; }
            double e2 = 0;
            for (int i = 0; i < L; i++) { double sc = cfg->abstol + cfg->reltol * fmax(fabs(z[i]), fabs(zn[i])); e2 += (errv[i] / sc) * (errv[i] / sc); }
            double EEst = sqrt(e2 / L);
            double q = step_factor_I(EEst, 1.0 / 3.0);
            if (EEst > 1.0) { h = hs / q; fsal_ok = 1; continue; }
            h = hs / q;
            memcpy(k, k1r, sizeof(double) * L); memcpy(k + L, k2r, sizeof(double) * L);
        }
        /* --- accepted step [t -> tn] --- */
        if (sa == SA_GAUSS) {
            /* IntegratingSumCallback: Gauss-Legendre over the step with the adjoint integrator's own
               interpolant for lam and the forward interpolant for y (gauss_adjoint.jl:745-759) */
            int ng = ros ? 1 : 3; const double* gx = ros ? GL1_X : GL3_X; const double* gw = ros ? GL1_W : GL3_W;
            for (int j = 0; j < ng; j++) {
                double tj = 0.5 * (tn - t) * gx[j] + 0.5 * (tn + t);
                double th = (tj - t) / hs;
                if (!ros) tsit5_dense(d, th, hs, z, k, lamq);
                else { double c1 = th * (1 - th) / (1 - 2 * ROS_D), c2 = th * (th - 2 * ROS_D) / (1 - 2 * ROS_D);
                       for (int i = 0; i < d; i++) lamq[i] = z[i] + hs * (c1 * k[i] + c2 * k[L + i]); }
                dense_eval(sol, tj, 0, ybuf, NULL);                        /* sol(y,t) */
                F->vjp(ybuf, p, tj, lamq, dlq, integ, &F->ctx);           /* vec_pjac! */
                for (int q = 0; q < P; q++) acc[q] += (0.5 * (tn - t)) * gw[j] * (-integ[q]);   /* out = -F'lam; scale (t-tprev)/2 */
            }
        }
        if (sa == SA_GAUSSKRONROD) {
            gkstep_ctx gc = {F, p, sol, ros, d, L, t, hs, z, k, ybuf, lamq, dlq};
            integrate_gk(gkstep_node, &gc, P, ros ? 1 : 3, t, tn, acc, 0);
        }
        if (have_adj) adjdense_push(&adj, t, hs, z, k);
        memcpy(z, zn, sizeof(double) * L);
        if (!ros) { memcpy(k, k + 6 * L, sizeof(double) * L); } else memcpy(f0, fnr, sizeof(double) * L);
        fsal_ok = 1;
        t = tn;
        if (!adaptive) h = -fabs(cfg->dt);
        APPLY_CKPT_IF_AT(t);
        APPLY_JUMP_IF_AT(t);
        APPLY_EVENT_IF_AT(t);
    }
    if (rc == 0) {
        for (int i = 0; i < d; i++) du0[i] = z[i];
        if (sa == SA_INTERPOLATING || sa == SA_BACKSOLVE) for (int q = 0; q < P; q++) dp[q] = z[d + q];
        else if (sa == SA_GAUSS || sa == SA_GAUSSKRONROD) for (int q = 0; q < P; q++) dp[q] = acc[q];
        else {
            /* QuadratureAdjoint interval loop (quadrature_adjoint.jl:537-616) */
            quad_ctx qc = {F, p, sol, &adj, ybuf, lamq, dlq};
            double* res = (double*)calloc(P, sizeof(double)), *part = (double*)malloc(sizeof(double) * P);
            if (K == 0) { oracle_quadgk(quad_integrand, &qc, P, t0, T, cfg->quad_abstol, cfg->quad_reltol, res); }
            else {
                if (ts[K - 1] != T) { oracle_quadgk(quad_integrand, &qc, P, ts[K - 1], T, cfg->quad_abstol, cfg->quad_reltol, part); for (int q = 0; q < P; q++) res[q] += part[q]; }
                for (int i = K - 2; i >= 0; i--) {
                    if (ts[i] == ts[i + 1]) continue;
                    oracle_quadgk(quad_integrand, &qc, P, ts[i], ts[i + 1], cfg->quad_abstol, cfg->quad_reltol, part);
                    for (int q = 0; q < P; q++) res[q] += part[q];
                }
                if (ts[0] != t0) { oracle_quadgk(quad_integrand, &qc, P, t0, ts[0], cfg->quad_abstol, cfg->quad_reltol, part); for (int q = 0; q < P; q++) res[q] += part[q]; }
            }
            for (int q = 0; q < P; q++) dp[q] = res[q];
            free(res); free(part);
        }
    }
    if (nrhs_out) *nrhs_out = ctx.nrhs;
    if (have_adj) adjdense_free(&adj);
    free(z); free(zn); free(tmp); free(k); free(ybuf);
    return rc;
}

/* =====================================================================================
 * SDE (diagonal noise): forward EM / EulerHeun on the dt grid with given increments dW[S][m],
 * BacksolveAdjoint reverse on the same grid with reversed noise (backsolve_adjoint.jl:274-419).
 * ===================================================================================== */
static void sde_forward_member(const oracle_cfg* cfg, const family_t* F, const double* p, const double* u0,
                               const double* dW /* [S][m] */, int S, double* us /* [(S+1)][d] */) {
    int d = F->d; double h = cfg->dt;
    double f[8], g[8], ub[8], fb[8], gb[8];
    memcpy(us, u0, sizeof(double) * d);
    for (int n = 0; n < S; n++) {
        const double* u = us + (size_t)n * d; double* un = us + (size_t)(n + 1) * d; double t = cfg->t0 + n * h;
        F->f(u, p, t, f, &F->ctx); fam_g(F, u, p, t, g);
        if (cfg->stepper == ST_EM) for (int i = 0; i < d; i++) un[i] = u[i] + h * f[i] + g[i] * dW[(size_t)n * d + i];
        else {
            for (int i = 0; i < d; i++) ub[i] = u[i] + h * f[i] + g[i] * dW[(size_t)n * d + i];
            F->f(ub, p, t + h, fb, &F->ctx); fam_g(F, ub, p, t + h, gb);
            for (int i = 0; i < d; i++) un[i] = u[i] + 0.5 * h * (f[i] + fb[i]) + 0.5 * (g[i] + gb[i]) * dW[(size_t)n * d + i];
        }
    }
}
/* drift and diffusion of the augmented reverse SDE, z = [lam; mu; y] */
static void sde_adj_drift(const family_t* F, const double* p, int ito, double t, const double* z, double* dz) {
    int d = F->d, P = F->P; const double* y = z + d + P;
    (ito ? F->vjp_ito : F->vjp)(y, p, t, z, dz, dz + d, &F->ctx);
    for (int i = 0; i < d + P; i++) dz[i] = -dz[i];
    (ito ? F->f_ito : F->f)(y, p, t, dz + d + P, &F->ctx);
}
/* diffusion applied to increments dWr[m]: returns the increment vector sum_i G[:,i] dWr_i */
static void sde_adj_diffusion_apply(const family_t* F, const double* p, double t, const double* z, const double* dWr, double* out, double* dgm) {
    int d = F->d, P = F->P; const double* y = z + d + P; double dl[8], g[8];
    fam_gvjp(F, y, p, t, z, dl, dgm); fam_g(F, y, p, t, g);
    for (int q = 0; q < P; q++) out[d + q] = 0;
    for (int i = 0; i < d; i++) {
        out[i] = -dl[i] * dWr[i];                                         /* dlam diag slots, negated (:56) */
        for (int q = 0; q < P; q++) out[d + q] += -dgm[i * P + q] * dWr[i];  /* dgrad P x m block, negated (:57) */
        out[d + P + i] = g[i] * dWr[i];                                    /* dy diag slots */
    }
}
static int adjoint_sde_member(const oracle_cfg* cfg, const family_t* F, const double* p, const double* us, const double* dW, int S,
                              const double* ts, const double* dL, double* du0, double* dp) {
    const int d = F->d, P = F->P, L = 2 * d + P, K = cfg->K;
    /* InterpolatingAdjoint (src/interpolating_adjoint.jl:453-613): z = [lam; mu], y(t) = sol(t) from the saved forward
     * solution (the reverse solve steps on the forward grid, src/sensitivity_interface.jl:484-486, so y is the stored
     * u_n), drift = sol.prob.f WITHOUT the Ito transformation (:525-533).  BacksolveAdjoint: z = [lam; mu; y], Ito ->
     * transformed drift (backsolve_adjoint.jl:327-345).  Both share this loop; for Interpolating the y slots are
     * overwritten from the forward solution before every drift/diffusion evaluation. */
    const int interp = (cfg->sensealg == SA_INTERPOLATING);
    const int ito = (cfg->stepper == ST_EM) && !interp;
    double h = cfg->dt;
    double* z = (double*)calloc(L, sizeof(double)), *a = (double*)malloc(sizeof(double) * L), *b = (double*)malloc(sizeof(double) * L);
    double* zb = (double*)malloc(sizeof(double) * L), *a2 = (double*)malloc(sizeof(double) * L), *b2 = (double*)malloc(sizeof(double) * L);
    double* dgm = (double*)malloc(sizeof(double) * d * P); double dWr[8], gu[8];
    memcpy(z + d + P, us + (size_t)S * d, sizeof(double) * d);
    int cur = K - 1;
    for (int n = S; n >= 0; n--) {
        double t = cfg->t0 + n * h; if (n == S) t = cfg->t1;
        /* callbacks at grid point n: checkpoint reset (y <- sol(t)) then loss jump */
        int is_save = (cur >= 0 && fabs(ts[cur] - t) <= 1e-9 * fmax(1.0, fabs(t)));
        if (interp || (cfg->checkpointing && (cfg->backsolve_ckpt_every_step || is_save))) memcpy(z + d + P, us + (size_t)n * d, sizeof(double) * d);
        if (is_save) {
            /* no_start skips the jump of the first save time for every sensealg but Backsolve (src/adjoint_common.jl:761) */
            if (!(cfg->no_start && cur == 0 && interp)) {
                cost_grad(cfg, dL ? dL + (size_t)cur * d : NULL, z + d + P, gu);
                for (int i = 0; i < d; i++) z[i] += gu[i];
            }
            cur--;
        }
        if (n == 0) break;
        /* reverse step n -> n-1: dt_rev = -h, dW_rev = W(t_{n-1}) - W(t_n) = -dW_{n-1} */
        for (int i = 0; i < d; i++) dWr[i] = -dW[(size_t)(n - 1) * d + i];
        sde_adj_drift(F, p, ito, t, z, a);
        sde_adj_diffusion_apply(F, p, t, z, dWr, b, dgm);
        if (cfg->stepper == ST_EM) for (int i = 0; i < L; i++) z[i] = z[i] - h * a[i] + b[i];
        else {
            for (int i = 0; i < L; i++) zb[i] = z[i] - h * a[i] + b[i];
            if (interp) memcpy(zb + d + P, us + (size_t)(n - 1) * d, sizeof(double) * d);      /* y(t_{n-1}) = sol(t_{n-1}) */
            sde_adj_drift(F, p, ito, t - h, zb, a2);
            sde_adj_diffusion_apply(F, p, t - h, zb, dWr, b2, dgm);
            for (int i = 0; i < L; i++) z[i] = z[i] - 0.5 * h * (a[i] + a2[i]) + 0.5 * (b[i] + b2[i]);
        }
    }
    for (int i = 0; i < d; i++) du0[i] = z[i];
    for (int q = 0; q < P; q++) dp[q] = z[d + q];
    free(z); free(a); free(b); free(zb); free(a2); free(b2); free(dgm);
    return 0;
}

/* =====================================================================================
 * Public entry points (ctypes).  Layouts match the C ABI of the product (trajectory-minor SoA):
 *   u0[d][N], p[P] or [P][N], saved[K][d][N], dLdu[K][d][N], du0[d][N], dp[P] or [P][N], dW[S][m][N]
 * ===================================================================================== */
static int is_sde(const oracle_cfg* c) { return c->stepper == ST_EM || c->stepper == ST_EULER_HEUN; }

static int forward_dense_member(const oracle_cfg* cfg, const family_t* F, const double* p, const double* u0, dense_t* S) {
    switch (cfg->stepper) {
    case ST_TSIT5_FIXED: forward_tsit5_fixed(F, p, u0, cfg->t0, cfg->t1, cfg->dt, S, cfg); return 0;
    case ST_TSIT5_ADAPTIVE: return forward_tsit5_adaptive(F, p, u0, cfg->t0, cfg->t1, cfg->abstol, cfg->reltol, cfg->dt, S, cfg);
    case ST_ROSENBROCK23: return forward_ros23(F, p, u0, cfg->t0, cfg->t1, cfg->abstol, cfg->reltol, S);
    default: return -5;
    }
}

/* One full gradient evaluation for the ensemble: forward dense solve, primal at saveat, reverse adjoint,
 * reduction of dp over members when p is shared.  `saved` and `dLdu` may be NULL (COST_AFFINE needs no dLdu).
 * steps_out[N] (optional) receives the number of forward steps per member. */
int oracle_ensemble_gradient(const oracle_cfg* cfg, const double* saveat, const double* u0, const double* p,
                             const double* dW, const double* dLdu, double* saved, double* du0, double* dp,
                             int32_t* steps_out, int nthreads) {
    family_t F; int rc = family_init(&F, cfg); if (rc) return rc;
    const int d = F.d, P = F.P, K = cfg->K; const int64_t N = cfg->N;
    int S = 0;
    if (is_sde(cfg)) { S = (int)llround((cfg->t1 - cfg->t0) / cfg->dt); if (cfg->sensealg != SA_BACKSOLVE && cfg->sensealg != SA_INTERPOLATING) return -6; }
    int err = 0;
    double* dp_members = (double*)calloc((size_t)N * P, sizeof(double));
#ifdef _OPENMP
    if (nthreads > 0) omp_set_num_threads(nthreads);
#endif
#pragma omp parallel for schedule(static)
    for (int64_t i = 0; i < N; i++) {
        double* pm = (double*)malloc(sizeof(double) * (P > 0 ? P : 1)), um[8], du[8];
        double* dpm = dp_members + (size_t)i * P;
        for (int q = 0; q < P; q++) pm[q] = cfg->shared_p ? p[q] : p[(size_t)q * N + i];
        for (int j = 0; j < d; j++) um[j] = u0[(size_t)j * N + i];
        double* dLm = NULL;
        int r = 0;
        if (!is_sde(cfg)) {
            dense_t sol;
            /* continuous callback: the forward solve FINDS this member's event times; the reverse pass sees them as a
             * member-local event list (times, effective affine affect) */
            cc_events found = {0, 0, NULL, NULL, NULL};
            oracle_cfg mcfg = *cfg;
            if (cfg->cc_on) {
                if (cfg->stepper != ST_TSIT5_ADAPTIVE) r = -12;
                else r = forward_tsit5_adaptive_cc(&F, pm, um, cfg->t0, cfg->t1, cfg->abstol, cfg->reltol, cfg->dt, &sol, cfg, &found);
                mcfg.n_events = found.n; mcfg.ev_times = found.t; mcfg.ev_scale = found.scale; mcfg.ev_shift = found.shift;
                mcfg.ev_pscale = NULL; mcfg.ev_pshift = NULL; mcfg.ev_acomp = NULL;
            } else
            r = forward_dense_member(cfg, &F, pm, um, &sol);
            const oracle_cfg* cfg_m = &mcfg;
            if (r == 0) {
                if (steps_out) steps_out[i] = sol.n;
                double y[8];
                if (saved) for (int k = 0; k < K; k++) {
                    int at_ev = 0;
                    for (int e = 0; e < cfg_m->n_events; e++) if (cfg_m->ev_times[e] == saveat[k]) at_ev = 1;
                    dense_eval(&sol, saveat[k], at_ev, y, NULL);
                    for (int j = 0; j < d; j++) saved[((size_t)k * d + j) * N + i] = y[j]; }
                if (du0) {
                    if (cfg->cost_kind == COST_EXPLICIT) {
                        dLm = (double*)malloc(sizeof(double) * K * d);
                        for (int k = 0; k < K; k++) for (int j = 0; j < d; j++) dLm[k * d + j] = dLdu[((size_t)k * d + j) * N + i];
                    }
                    r = adjoint_ode_member(cfg_m, &F, pm, &sol, saveat, dLm, du, dpm, NULL);
                }
            }
            if (steps_out && cfg->cc_on) steps_out[i] = sol.n;
            dense_free(&sol); free(found.t); free(found.scale); free(found.shift);
        } else {
            double* us = (double*)malloc(sizeof(double) * (size_t)(S + 1) * d);
            double* dWm = (double*)malloc(sizeof(double) * (size_t)S * d);
            for (int n = 0; n < S; n++) for (int j = 0; j < d; j++) dWm[(size_t)n * d + j] = dW[((size_t)n * d + j) * N + i];
            sde_forward_member(cfg, &F, pm, um, dWm, S, us);
            if (steps_out) steps_out[i] = S;
            if (saved) for (int k = 0; k < K; k++) {
                int n = (int)llround((saveat[k] - cfg->t0) / cfg->dt);
                for (int j = 0; j < d; j++) saved[((size_t)k * d + j) * N + i] = us[(size_t)n * d + j];
            }
            if (du0) {
                if (cfg->cost_kind == COST_EXPLICIT) {
                    dLm = (double*)malloc(sizeof(double) * K * d);
                    for (int k = 0; k < K; k++) for (int j = 0; j < d; j++) dLm[k * d + j] = dLdu[((size_t)k * d + j) * N + i];
                }
                r = adjoint_sde_member(cfg, &F, pm, us, dWm, S, saveat, dLm, du, dpm);
            }
            free(us); free(dWm);
        }
        if (r == 0 && du0) for (int j = 0; j < d; j++) du0[(size_t)j * N + i] = du[j];
        if (r == 0 && du0 && (cfg->dgdp_c || cfg->dgdp_e || cfg->cdgdp_c || cfg->cdgdp_e)) {
            /* parameter part of the cost family: dgdp_discrete = c .* p + e joins the gradient at every save time whose jump is
             * applied (ReverseLossCallback, src/adjoint_common.jl:771-783; quadrature_adjoint.jl:547-553, 601-605), dgdp_continuous
             * integrates to (T - t0)(cc .* p + ce) (accumulate_cost!, src/derivative_wrappers.jl:1411-1442) */
            int njump = K;
            if (cfg->no_start && cfg->sensealg != SA_BACKSOLVE && K > 0 && saveat[0] == cfg->t0) njump--;
            for (int q = 0; q < P; q++) {
                dpm[q] += njump * ((cfg->dgdp_c ? cfg->dgdp_c[q] * pm[q] : 0.0) + (cfg->dgdp_e ? cfg->dgdp_e[q] : 0.0));
                if (cfg->cont_cost) dpm[q] += (cfg->t1 - cfg->t0) * ((cfg->cdgdp_c ? cfg->cdgdp_c[q] * pm[q] : 0.0) + (cfg->cdgdp_e ? cfg->cdgdp_e[q] : 0.0));
            }
        }
        if (r) {
#pragma omp atomic write
            err = r;
        }
        free(dLm); free(pm);
    }
    if (du0 && dp) {
        if (cfg->shared_p) {
            /* fixed-order pairwise (tree) sum over members: the reduction the outer AD does (ensembles.jl:22-31) */
            for (int q = 0; q < P; q++) {
                int64_t n = N; double* w = (double*)malloc(sizeof(double) * N);
                for (int64_t i = 0; i < N; i++) w[i] = dp_members[(size_t)i * P + q];
                while (n > 1) { int64_t hlf = (n + 1) / 2; for (int64_t i = 0; i + hlf < n; i++) w[i] += w[i + hlf]; n = hlf; }
                dp[q] = w[0]; free(w);
            }
        } else for (int64_t i = 0; i < N; i++) for (int q = 0; q < P; q++) dp[(size_t)q * N + i] = dp_members[(size_t)i * P + q];
    }
    free(dp_members);
    return err;
}

/* scalar loss of COST_AFFINE, L = sum_k sum_j (a/2 u^2 + b u), and explicit-cotangent-free forward solve:
 * used by the tests to differentiate THROUGH the solver by finite differences (the ForwardDiff relation). */
typedef struct { const dense_t* sol; const oracle_cfg* cfg; int d; double* y; } gint_ctx;
static void g_integrand(double t, double* out, void* c) {
    gint_ctx* x = (gint_ctx*)c; double s = 0;
    dense_eval(x->sol, t, 0, x->y, NULL);
    for (int j = 0; j < x->d; j++) s += 0.5 * CONT_A(x->cfg, j) * x->y[j] * x->y[j] + CONT_B(x->cfg, j) * x->y[j];
    out[0] = s;
}
/* integral of the continuous cost along one member's dense forward solution (quadgk per step, tight tolerance) */
int oracle_continuous_loss(const oracle_cfg* cfg, const double* u0, const double* p, double* out_members, int nthreads) {
    family_t F; int rc = family_init(&F, cfg); if (rc) return rc;
    const int d = F.d, P = F.P; const int64_t N = cfg->N;
#ifdef _OPENMP
    if (nthreads > 0) omp_set_num_threads(nthreads);
#endif
#pragma omp parallel for schedule(static)
    for (int64_t i = 0; i < N; i++) {
        double pm[16], um[8], y[8], part; dense_t sol;
        for (int q = 0; q < P && q < 16; q++) pm[q] = cfg->shared_p ? p[q] : p[(size_t)q * N + i];
        for (int j = 0; j < d; j++) um[j] = u0[(size_t)j * N + i];
        forward_dense_member(cfg, &F, pm, um, &sol);
        gint_ctx gc = {&sol, cfg, d, y};
        double tot = 0;
        for (int n = 0; n < sol.n; n++) { oracle_quadgk(g_integrand, &gc, 1, sol.t[n], sol.t[n + 1], 1e-14, 1e-13, &part); tot += part; }
        /* parameter part of the running cost: constant along the trajectory */
        for (int q = 0; q < P && q < 16; q++) tot += (cfg->t1 - cfg->t0) * ((cfg->cdgdp_c ? 0.5 * cfg->cdgdp_c[q] * pm[q] * pm[q] : 0.0) + (cfg->cdgdp_e ? cfg->cdgdp_e[q] * pm[q] : 0.0));
        out_members[i] = tot;
        dense_free(&sol);
    }
    return 0;
}

int oracle_ensemble_loss(const oracle_cfg* cfg, const double* saveat, const double* u0, const double* p,
                         const double* dW, double* loss_members /* [N] */, int nthreads) {
    const int d = cfg->d, K = cfg->K; const int64_t N = cfg->N;
    double* saved = (double*)malloc(sizeof(double) * (size_t)K * d * N);
    int rc = oracle_ensemble_gradient(cfg, saveat, u0, p, dW, NULL, saved, NULL, NULL, NULL, nthreads);
    for (int64_t i = 0; i < N; i++) {
        double s = 0;
        for (int k = 0; k < K; k++) for (int j = 0; j < d; j++) { double u = saved[((size_t)k * d + j) * N + i]; s += 0.5 * COST_A(cfg, j) * u * u + COST_B(cfg, j) * u; }
        for (int q = 0; q < cfg->P && (cfg->dgdp_c || cfg->dgdp_e); q++) {          /* parameter part, once per save time */
            const double pq = cfg->shared_p ? p[q] : p[(size_t)q * N + i];
            s += K * ((cfg->dgdp_c ? 0.5 * cfg->dgdp_c[q] * pq * pq : 0.0) + (cfg->dgdp_e ? cfg->dgdp_e[q] * pq : 0.0));
        }
        loss_members[i] = s;
    }
    free(saved);
    if (rc == 0 && cfg->cont_cost) {
        double* ci = (double*)malloc(sizeof(double) * N);
        rc = oracle_continuous_loss(cfg, u0, p, ci, nthreads);
        for (int64_t i = 0; i < N; i++) loss_members[i] += ci[i];
        free(ci);
    }
    return rc;
}

/* direct access to the RHS families for unit tests of the hand VJPs */
int oracle_family_eval(const oracle_cfg* cfg, int ito, const double* u, const double* p, const double* lam,
                       double* f_out, double* jtl_out, double* ftl_out) {
    family_t F; int rc = family_init(&F, cfg); if (rc) return rc;
    (ito ? F.f_ito : F.f)(u, p, 0.0, f_out, &F.ctx);
    (ito ? F.vjp_ito : F.vjp)(u, p, 0.0, lam, jtl_out, ftl_out, &F.ctx);
    return 0;
}
/* the event list of ONE member's hybrid forward solve (continuous callback): times[max_events], the states left and right of
 * every event, uminus / uplus [max_events][d].  Returns the number of events (all of them counted, the first max_events
 * stored) or a negative error.  Unit tests of the event location (test/Callbacks2/continuous_vs_discrete.jl:19-21). */
int oracle_event_list(const oracle_cfg* cfg, const double* u0, const double* p, int max_events, double* times,
                      double* uminus, double* uplus) {
    family_t F; int rc = family_init(&F, cfg); if (rc) return rc;
    if (!cfg->cc_on || cfg->stepper != ST_TSIT5_ADAPTIVE) return -12;
    dense_t sol; cc_events found = {0, 0, NULL, NULL, NULL};
    rc = forward_tsit5_adaptive_cc(&F, p, u0, cfg->t0, cfg->t1, cfg->abstol, cfg->reltol, cfg->dt, &sol, cfg, &found);
    int n = rc ? rc : found.n;
    for (int e = 0; rc == 0 && e < found.n && e < max_events; e++) {
        times[e] = found.t[e];
        if (uminus) dense_eval(&sol, found.t[e], 0, uminus + (size_t)e * F.d, NULL);
        if (uplus) dense_eval(&sol, found.t[e], 1, uplus + (size_t)e * F.d, NULL);
    }
    dense_free(&sol); free(found.t); free(found.scale); free(found.shift);
    return n;
}
int oracle_sizeof_cfg(void) { return (int)sizeof(oracle_cfg); }
