// api.cu -- C ABI (include/b200adj.h) of the H100-native (sm_90a) ensemble continuous-adjoint engine.
// Handle management, validation, host<->device staging; kernel dispatch goes through handle.h into disp_*.cu.
// No torch types, no CPU fallback.
#include <dlfcn.h>

#include "handle.h"

using namespace b200adj;
namespace {

thread_local std::string g_create_error;

// registered plug-in families (append-only; a registration is as global as the dlopen behind it)
std::vector<const FamilyVTable*>& family_registry() { static std::vector<const FamilyVTable*> r; return r; }

int fam_dims(const b200adj_cfg& c, int* d, int* P, int* m) {
    if (const FamilyVTable* vt = family_lookup(c.rhs_family)) { *d = vt->d; *P = vt->P; *m = 0; return 0; }
    switch (c.rhs_family) {
    case B200ADJ_FAM_LV: *d = 2; *P = 4; *m = 0; return 0;
    case B200ADJ_FAM_LORENZ: *d = 3; *P = 3; *m = 0; return 0;
    case B200ADJ_FAM_ROBERTSON: *d = 3; *P = 3; *m = 0; return 0;
    case B200ADJ_FAM_SDE_LV: *d = 2; *P = 6; *m = 2; return 0;
    case B200ADJ_FAM_SDE_LINEAR: *d = 2; *P = 2; *m = 2; return 0;
    case B200ADJ_FAM_BALL: *d = 2; *P = 2; *m = 0; return 0;
    case B200ADJ_FAM_RELAX: *d = 1; *P = 2; *m = 0; return 0;
    case B200ADJ_FAM_MLP: if (c.mlp_hidden != MLP_H) return -1; *d = MLP_D; *P = MLP_P; *m = 0; return 0;
    default: return -1;
    }
}
}  // namespace

namespace b200adj {
// Tsit5 dense-output weights b_j(theta): quartics, expanded once in long double from the published factored form
// (Tsitouras 2011; SURVEY.md App. B) and evaluated by Horner.
void tsit5_weights(double th, double* w, double (*Rout)[4]) {
    typedef long double LD;
    static bool init = false;
    static double R[7][5];   // coefficients of theta^0..theta^4
    if (!init) {
        auto mul = [](const LD* a, int na, const LD* b, int nb, LD* out) {
            for (int i = 0; i < na + nb - 1; i++) out[i] = 0;
            for (int i = 0; i < na; i++) for (int j = 0; j < nb; j++) out[i + j] += a[i] * b[j];
        };
        LD t1[2] = {0, 1};
        {   LD a[2] = {-1.3299890189751412L, 1}, q[3] = {0.7139816917074209L, -1.4364028541716351L, 1}, x[3], y[5];
            mul(t1, 2, a, 2, x); mul(x, 3, q, 3, y);
            for (int i = 0; i < 5; i++) R[0][i] = (double)(-1.0530884977290216L * y[i]); }
        auto sq_quad = [&](int row, LD c, LD s, LD wq) {      // c * th^2 * (th^2 - s th + wq)
            R[row][0] = 0; R[row][1] = 0; R[row][2] = (double)(c * wq); R[row][3] = (double)(-c * s); R[row][4] = (double)c; };
        auto sq_roots = [&](int row, LD c, LD r1, LD r2) {    // c * (th - r1)(th - r2) * th^2
            R[row][0] = 0; R[row][1] = 0; R[row][2] = (double)(c * r1 * r2); R[row][3] = (double)(-c * (r1 + r2)); R[row][4] = (double)c; };
        sq_quad(1, 0.1017L, 2.1966568338249754L, 1.2949852507374631L);
        sq_quad(2, 2.490627285651252793L, 2.38535645472061657L, 1.57803468208092486L);
        sq_roots(3, -16.54810288924490272L, 1.21712927295533244L, 0.61620406037800089L);
        sq_roots(4, 47.37952196281928122L, 1.203071208372362603L, 0.658047292653547382L);
        sq_roots(5, -34.87065786149660974L, 1.2L, 0.666666666666666667L);
        sq_roots(6, 2.5L, 1.0L, 0.6L);
        init = true;
    }
    if (Rout) for (int j = 0; j < 7; j++) for (int m = 0; m < 4; m++) Rout[j][m] = R[j][m + 1];
    if (w) for (int j = 0; j < 7; j++) w[j] = (((R[j][4] * th + R[j][3]) * th + R[j][2]) * th + R[j][1]) * th + R[j][0];
}
}  // namespace b200adj

namespace {
// Step-size-scaled Tsit5 tables for one handle (passed to the kernels by value, i.e. through the constant bank).
void build_tsit5_tables(double h, Tsit5Tables* t) {
    const double A[7][6] = {
        {0},
        {0.161},
        {-0.008480655492356989, 0.335480655492357},
        {2.8971530571054935, -6.359448489975075, 4.3622954328695815},
        {5.325864828439257, -11.748883564062828, 7.4955393428898365, -0.09249506636175525},
        {5.86145544294642, -12.92096931784711, 8.159367898576159, -0.071584973281401, -0.028269050394068383},
        {0.09646076681806523, 0.01, 0.4798896504144996, 1.379008574103742, -3.290069515436081, 2.324710524099774}};
    const double C[7] = {0.0, 0.161, 0.327, 0.9, 0.9800255409045097, 1.0, 1.0};
    memset(t, 0, sizeof(*t));
    for (int s = 0; s < 7; s++) for (int j = 0; j < 6; j++) t->hA[s][j] = h * A[s][j];
    double w[7];
    for (int s = 1; s <= 4; s++) { tsit5_weights(1.0 - C[s], w); for (int j = 0; j < 7; j++) t->hBst[s - 1][j] = h * w[j]; }
    const double a = sqrt(0.6);
    const double thq[3] = {0.5 * (1.0 - a), 0.5, 0.5 * (1.0 + a)};
    for (int g = 0; g < 3; g++) { tsit5_weights(thq[g], w); for (int j = 0; j < 7; j++) t->hBq[g][j] = h * w[j]; }
    t->hGW[0] = 0.5 * h * (5.0 / 9.0); t->hGW[1] = 0.5 * h * (8.0 / 9.0); t->hGW[2] = 0.5 * h * (5.0 / 9.0);
}
T5aArgs t5a_args(Handle* h) {
    const b200adj_cfg& c = h->cfg;
    T5aArgs a;
    memset(&a, 0, sizeof(a));
    a.saveat = h->d_saveat; a.partials = h->d_partials; a.ticket = h->d_ticket;
    a.ft = h->r_ft; a.fu = h->r_fu; a.fk = h->r_fk; a.fn = h->r_fn;
    a.rrec = h->r_rrec; a.rend = h->r_rend; a.ftT = h->r_ftT; a.frecT = h->r_frecT; a.rn = h->r_rn;
    a.qseg = h->r_qseg; a.qkey = h->r_qkey; a.maxseg = h->maxseg;
    a.N = c.N; a.K = c.K; a.maxs = h->maxs; a.t0 = c.t0; a.t1 = c.t1; a.dt0 = c.dt; a.abstol = c.abstol; a.reltol = c.reltol;
    a.quad_abstol = c.quad_abstol; a.quad_reltol = c.quad_reltol;
    for (int j = 0; j < 4; j++) { a.cost_a[j] = h->cost_av[j]; a.cost_b[j] = h->cost_bv[j]; }
    a.flags = ((c.flags & B200ADJ_FLAG_NO_START) ? 1u : 0u) | ((c.flags & B200ADJ_FLAG_NO_CHECKPOINTING) ? 2u : 0u) |
              ((c.flags & B200ADJ_FLAG_CKPT_EVERY_STEP) ? 4u : 0u);
    const double A[7][6] = {
        {0},
        {0.161},
        {-0.008480655492356989, 0.335480655492357},
        {2.8971530571054935, -6.359448489975075, 4.3622954328695815},
        {5.325864828439257, -11.748883564062828, 7.4955393428898365, -0.09249506636175525},
        {5.86145544294642, -12.92096931784711, 8.159367898576159, -0.071584973281401, -0.028269050394068383},
        {0.09646076681806523, 0.01, 0.4798896504144996, 1.379008574103742, -3.290069515436081, 2.324710524099774}};
    const double C[7] = {0.0, 0.161, 0.327, 0.9, 0.9800255409045097, 1.0, 1.0};
    const double BT[7] = {-0.00178001105222577714, -0.0008164344596567469, 0.007880878010261995, -0.1447110071732629,
                          0.5823571654525552, -0.45808210592918697, 0.015151515151515152};
    memcpy(a.A, A, sizeof(A)); memcpy(a.C, C, sizeof(C)); memcpy(a.BT, BT, sizeof(BT));
    tsit5_weights(0.0, nullptr, a.R);
    if (h->fixed_dt) a.flags |= 16u;          // constant step, no error control (fixed-step Tsit5 on the dense framework)
    if (h->cont_on) { a.flags |= 8u; for (int j = 0; j < 4; j++) { a.cont_a[j] = h->cont_av[j]; a.cont_b[j] = h->cont_bv[j]; } }
    a.nev = h->nev; a.ev_t = h->d_ev_t; a.ev_s = h->d_ev_s; a.ev_c = h->d_ev_c; a.ev_ps = h->d_ev_ps; a.ev_pc = h->d_ev_pc;
    a.ev_ac = h->d_ev_ac; a.ev_ak = h->d_ev_ak; a.ev_af = h->d_ev_af;
    if (h->cc_on) {
        a.cc_on = 1; a.cc_idx = h->cc_idx; a.cc_dir = h->cc_dir; a.cc_pcomp = h->cc_pcomp; a.cc_pparam = h->cc_pparam; a.cc_maxev = h->cc_maxev;
        a.cc_level = h->cc_level; a.cc_psign = h->cc_psign; a.cc_t = h->d_cc_t; a.cc_n = h->d_cc_n;
        for (int j = 0; j < 4; j++) { a.cc_scale[j] = h->cc_scale[j]; a.cc_shift[j] = h->cc_shift[j]; }
        a.cc_lparam = h->cc_lparam; a.cc_lcoef = h->cc_lcoef; a.cc_acomp = h->cc_acomp; a.cc_aparam = h->cc_aparam; a.cc_acoef = h->cc_acoef;
        a.cc_qcomp = h->cc_qcomp; a.cc_qcoef = h->cc_qcoef;
    }
    return a;
}
RosArgs ros_args(Handle* h) {
    const b200adj_cfg& c = h->cfg;
    RosArgs a;
    memset(&a, 0, sizeof(a));
    a.saveat = h->d_saveat; a.partials = h->d_partials; a.ticket = h->d_ticket;
    a.ft = h->r_ft; a.fu = h->r_fu; a.fk = h->r_fk; a.fn = h->r_fn;
    a.rrec = h->r_rrec; a.rend = h->r_rend; a.ftT = h->r_ftT; a.frecT = h->r_frecT; a.rn = h->r_rn;
    a.qseg = h->r_qseg; a.qkey = h->r_qkey; a.maxseg = h->maxseg;
    a.N = c.N; a.K = c.K; a.maxs = h->maxs; a.t0 = c.t0; a.t1 = c.t1; a.abstol = c.abstol; a.reltol = c.reltol;
    a.quad_abstol = c.quad_abstol; a.quad_reltol = c.quad_reltol;
    for (int j = 0; j < 4; j++) { a.cost_a[j] = h->cost_av[j]; a.cost_b[j] = h->cost_bv[j]; }
    a.flags = ((c.flags & B200ADJ_FLAG_NO_START) ? 1u : 0u) | ((c.flags & B200ADJ_FLAG_NO_CHECKPOINTING) ? 2u : 0u) |
              ((c.flags & B200ADJ_FLAG_CKPT_EVERY_STEP) ? 4u : 0u);
    return a;
}
void free_all(Handle* h) {
    cudaSetDevice(h->cfg.device);
    cudaFree(h->r_ft); cudaFree(h->r_fu); cudaFree(h->r_fk); cudaFree(h->r_rrec); cudaFree(h->r_rend); cudaFree(h->r_ftT); cudaFree(h->r_frecT);
    cudaFree(h->d_saveat); cudaFree(h->r_fn); cudaFree(h->r_rn); cudaFree(h->r_qseg); cudaFree(h->r_qkey);
    cudaFree(h->d_kst); cudaFree(h->d_adj_dense); cudaFree(h->d_trace); cudaFree(h->d_ckpt); cudaFree(h->d_noise); cudaFree(h->d_partials); cudaFree(h->d_ticket); cudaFree(h->d_save_of_step); cudaFree(h->d_fwd_save_of_step); cudaFree(h->d_fwd_saveat);
    cudaFree(h->s_u0); cudaFree(h->s_p); cudaFree(h->s_saved); cudaFree(h->s_dLdu); cudaFree(h->s_du0); cudaFree(h->s_dp); cudaFree(h->s_dW);
    cudaFree(h->d_cc_t); cudaFree(h->d_cc_n);
    cudaFree(h->s_status); cudaFree(h->d_event_of_step); cudaFree(h->d_ev_ac); cudaFree(h->d_ev_ak); cudaFree(h->d_ev_af); cudaFree(h->d_ev_t); cudaFree(h->d_ev_s); cudaFree(h->d_ev_c); cudaFree(h->d_ev_ps); cudaFree(h->d_ev_pc);
    if (h->own_stream) cudaStreamDestroy(h->own_stream);
}

}  // namespace

namespace {
// dp += coef_c .* p + coef_e per member (shared parameters: N times, once)
struct DgdpArgs { double c[8], e[8]; const void* p; void* dp; int64_t N; int32_t P, shared_p, f32; };
__global__ void dgdp_add_kernel(DgdpArgs g) {
    const int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (g.shared_p) {
        if (i != 0) return;
        for (int q = 0; q < g.P; q++) {
            if (g.f32) { float* dp = (float*)g.dp; const float* p = (const float*)g.p; dp[q] = (float)((double)dp[q] + (double)g.N * (g.c[q] * (double)p[q] + g.e[q])); }
            else { double* dp = (double*)g.dp; const double* p = (const double*)g.p; dp[q] += (double)g.N * (g.c[q] * p[q] + g.e[q]); }
        }
        return;
    }
    if (i >= g.N) return;
    for (int q = 0; q < g.P; q++) {
        if (g.f32) { float* dp = (float*)g.dp; const float* p = (const float*)g.p; dp[(int64_t)q * g.N + i] += (float)(g.c[q] * (double)p[(int64_t)q * g.N + i] + g.e[q]); }
        else { double* dp = (double*)g.dp; const double* p = (const double*)g.p; dp[(int64_t)q * g.N + i] += g.c[q] * p[(int64_t)q * g.N + i] + g.e[q]; }
    }
}
}  // namespace

namespace b200adj {
const FamilyVTable* family_lookup(int id) {
    auto& r = family_registry();
    const int k = id - B200ADJ_FAM_USER_BASE_ID;
    return (k >= 0 && k < (int)r.size()) ? r[k] : nullptr;
}
}  // namespace b200adj

namespace b200adj {
// QuadratureAdjoint on an adaptive handle: the dense reverse solution, the member-major copy of the forward one and the
// quadgk scratch are only needed by this sensealg -- allocate them at its first reverse pass
int ensure_quad_buffers(Handle* h) {
    if (h->r_rrec) return B200ADJ_OK;
    const b200adj_cfg& c = h->cfg;
    const size_t N = (size_t)c.N, MS = (size_t)h->maxs, e = sizeof(double);
    const size_t RWP = quad_pad(3 + (1 + h->nk) * c.d), FWP = quad_pad((1 + h->nk) * c.d + 3);
    const bool t5a = h->nk == 7;      // adaptive Tsit5: the forward dense solution is member-major from the start (allocated at create)
    if (cudaMalloc(&h->r_rrec, N * MS * RWP * e) != cudaSuccess || cudaMalloc(&h->r_rend, N * MS * e) != cudaSuccess ||
        (!t5a && (cudaMalloc(&h->r_ftT, N * (MS + 1) * e) != cudaSuccess || cudaMalloc(&h->r_frecT, N * MS * FWP * e) != cudaSuccess)) ||
        cudaMalloc(&h->r_qseg, quad_seg_doubles(c.P, h->maxseg, h->qgrid) * e) != cudaSuccess ||
        cudaMalloc(&h->r_qkey, (size_t)h->qgrid * QUAD_WARPS * h->maxseg * e) != cudaSuccess) {
        cudaGetLastError();
        h->err = "out of device memory for the QuadratureAdjoint buffers (dense reverse solution: N * max_steps records)";
        return B200ADJ_ERR_OOM;
    }
    return B200ADJ_OK;
}
}  // namespace b200adj

extern "C" {

uint32_t b200adj_version(void) { return 0x000201u; }
uint32_t b200adj_sizeof_cfg(void) { return (uint32_t)sizeof(b200adj_cfg); }

const char* b200adj_last_error(void* handle) {
    if (!handle) return g_create_error.c_str();
    return ((Handle*)handle)->err.c_str();
}

int32_t b200adj_create(const b200adj_cfg* cfg, void** handle) {
    if (!cfg || !handle) { g_create_error = "null cfg/handle"; return B200ADJ_ERR_INVALID; }
    *handle = nullptr;
    int ndev = 0;
    if (cudaGetDeviceCount(&ndev) != cudaSuccess || ndev == 0 || cfg->device < 0 || cfg->device >= ndev) {
        g_create_error = "no usable CUDA device (libb200adj has no CPU fallback)";
        return B200ADJ_ERR_NO_DEVICE;
    }
    int d, P, m;
    if (fam_dims(*cfg, &d, &P, &m)) { g_create_error = "rhs_family not built (MLP / unknown)"; return B200ADJ_ERR_UNSUPPORTED; }
    if (cfg->d != d || cfg->P != P) { g_create_error = "cfg.d / cfg.P do not match rhs_family"; return B200ADJ_ERR_INVALID; }
    // Fixed-step Tsit5 with save times OFF the dt grid (or B200ADJ_FLAG_DENSE_FORWARD): the reference interpolates the dense
    // forward solution at saveat (src/concrete_solve.jl:752-769) and the jump times become tstops of the fixed-dt reverse
    // solve, whose grid then shifts.  That needs the dense forward solution (k1..k7 per step) and general-theta lookups: the
    // per-member framework of the adaptive steppers run with a constant step (t5a kernels, T5A_FLAG_FIXED_DT).
    bool dense_fixed = false;
    if (cfg->stepper == B200ADJ_ST_TSIT5_FIXED && cfg->dtype == B200ADJ_F64 && cfg->rhs_family != B200ADJ_FAM_MLP && cfg->dt > 0) {
        dense_fixed = (cfg->flags & B200ADJ_FLAG_DENSE_FORWARD) != 0;
        for (int k = 0; k < cfg->K && cfg->saveat && !dense_fixed; k++) {
            const long long n = llround((cfg->saveat[k] - cfg->t0) / cfg->dt);
            if (fabs(cfg->t0 + n * cfg->dt - cfg->saveat[k]) > 1e-9 * fmax(1.0, fabs(cfg->saveat[k]))) dense_fixed = true;
        }
        if (dense_fixed && cfg->checkpoint_every > 1) { g_create_error = "checkpoint_every > 1 needs save times on the dt grid"; return B200ADJ_ERR_UNSUPPORTED; }
    }
    const bool t5a = cfg->stepper == B200ADJ_ST_TSIT5_ADAPTIVE || dense_fixed;
    const bool ros = cfg->stepper == B200ADJ_ST_ROSENBROCK23 || t5a;      // per-member adaptive framework
    if (cfg->N <= 0 || cfg->K < 0 || (cfg->K > 0 && !cfg->saveat) || (!ros && !(cfg->dt > 0)) || !(cfg->t1 > cfg->t0)) {
        g_create_error = "bad N/K/saveat/dt/tspan"; return B200ADJ_ERR_INVALID; }
    const bool mlp = cfg->rhs_family == B200ADJ_FAM_MLP;
    // F32: the MLP family and the fixed-step Tsit5 ODE path of LV / Lorenz (the fp32 throughput variant, SURVEY.md 8d C2)
    const bool f32_ode = cfg->dtype == B200ADJ_F32 && cfg->stepper == B200ADJ_ST_TSIT5_FIXED &&
                         (cfg->rhs_family == B200ADJ_FAM_LV || cfg->rhs_family == B200ADJ_FAM_LORENZ);
    if (f32_ode && cfg->sensealg == B200ADJ_SA_QUADRATURE) { g_create_error = "F32: Interpolating / Gauss / Backsolve (QuadratureAdjoint is F64 only)"; return B200ADJ_ERR_UNSUPPORTED; }
    if (cfg->dtype != B200ADJ_F64 && !f32_ode && !(mlp && (cfg->dtype == B200ADJ_F32 || cfg->dtype == B200ADJ_BF16_F32ACC))) {
        g_create_error = "dtype: F64 (all families), F32 (MLP; LV / Lorenz with fixed-step Tsit5), BF16_F32ACC (MLP) are built"; return B200ADJ_ERR_UNSUPPORTED; }
    if (mlp && (cfg->stepper != B200ADJ_ST_TSIT5_FIXED || (cfg->sensealg != B200ADJ_SA_INTERPOLATING && cfg->sensealg != B200ADJ_SA_GAUSS) || !cfg->shared_p)) {
        g_create_error = "MLP family: InterpolatingAdjoint / GaussAdjoint + fixed-step Tsit5 + shared parameters are built"; return B200ADJ_ERR_UNSUPPORTED; }
    if (cfg->cost_kind != B200ADJ_COST_EXPLICIT && cfg->cost_kind != B200ADJ_COST_AFFINE) { g_create_error = "bad cost_kind"; return B200ADJ_ERR_INVALID; }
    const bool sde = is_sde(*cfg);
    if (sde) {
        if (m == 0) { g_create_error = "SDE stepper needs an SDE family"; return B200ADJ_ERR_INVALID; }
        if (cfg->sensealg != B200ADJ_SA_BACKSOLVE && cfg->sensealg != B200ADJ_SA_INTERPOLATING) { g_create_error = "SDE: BacksolveAdjoint / InterpolatingAdjoint are built"; return B200ADJ_ERR_UNSUPPORTED; }
    } else {
        if (m != 0) { g_create_error = "ODE stepper with an SDE family"; return B200ADJ_ERR_INVALID; }
        if (cfg->sensealg < 0 || cfg->sensealg > 4) { g_create_error = "bad sensealg"; return B200ADJ_ERR_INVALID; }
        if (cfg->sensealg == B200ADJ_SA_GAUSSKRONROD && (mlp || cfg->dtype != B200ADJ_F64)) { g_create_error = "GaussKronrodAdjoint: F64, named ODE families"; return B200ADJ_ERR_UNSUPPORTED; }
        if (cfg->stepper != B200ADJ_ST_TSIT5_FIXED && !ros) { g_create_error = "stepper not built on device yet"; return B200ADJ_ERR_UNSUPPORTED; }
        if (ros && !dense_fixed && !(cfg->abstol > 0 && cfg->reltol > 0)) { g_create_error = "adaptive steppers need abstol, reltol > 0"; return B200ADJ_ERR_INVALID; }
        if (ros && mlp) { g_create_error = "MLP family: fixed-step Tsit5 only"; return B200ADJ_ERR_UNSUPPORTED; }
    }
    if (cfg->rhs_family == B200ADJ_FAM_RELAX && !t5a) { g_create_error = "Relax family: Tsit5 on the per-member dense framework (adaptive, or fixed step with B200ADJ_FLAG_DENSE_FORWARD)"; return B200ADJ_ERR_UNSUPPORTED; }
    if (cfg->rhs_family == B200ADJ_FAM_BALL && !t5a) { g_create_error = "BouncingBall family: Tsit5 on the per-member dense framework (adaptive, or fixed step with B200ADJ_FLAG_DENSE_FORWARD)"; return B200ADJ_ERR_UNSUPPORTED; }
    if (ros) {
        // adaptive path: save times are arbitrary ascending points of [t0, t1] (tstops of the reverse solve)
        for (int k = 0; k < cfg->K; k++) {
            if (cfg->saveat[k] < cfg->t0 || cfg->saveat[k] > cfg->t1 || (k > 0 && !(cfg->saveat[k] > cfg->saveat[k - 1]))) {
                g_create_error = "saveat must be ascending inside [t0, t1]"; return B200ADJ_ERR_INVALID; }
        }
        Handle* h = new Handle();
        h->cfg = *cfg; h->cfg.m = 0; h->adaptive = true; h->nk = t5a ? 7 : 2; h->fixed_dt = dense_fixed;
        h->saveat.assign(cfg->saveat, cfg->saveat + cfg->K);
        h->cfg.saveat = h->saveat.data();
        h->maxs = cfg->max_steps > 0 ? cfg->max_steps : 4096;      // per-member step capacity (forward and dense reverse)
        if (dense_fixed) {
            // constant step: S forward steps; the reverse solve adds at most one clipped step per tstop (save times, events)
            const long long S_ = llround((cfg->t1 - cfg->t0) / cfg->dt);
            if (S_ < 1 || fabs(S_ * cfg->dt - (cfg->t1 - cfg->t0)) > 1e-9 * fmax(1.0, fabs(cfg->t1 - cfg->t0))) {
                g_create_error = "(t1-t0) is not a whole number of dt steps"; delete h; return B200ADJ_ERR_UNSUPPORTED; }
            const long long need = S_ + cfg->K + 64;
            if (h->maxs < need) h->maxs = (int)(((need + 31) / 32) * 32);
        }
        h->block = cfg->block_threads ? cfg->block_threads : 128;
        if (h->block < 32 || h->block > 256 || (h->block % 32)) { g_create_error = "block_threads must be a multiple of 32 in [32, 256] for Rosenbrock23"; delete h; return B200ADJ_ERR_INVALID; }
        h->grid = (int)((cfg->N + h->block - 1) / h->block);
#define CREATE_TRY(expr)                                                                         \
        do { cudaError_t _e = (expr); if (_e != cudaSuccess) {                                   \
            g_create_error = std::string(#expr) + ": " + cudaGetErrorString(_e);                 \
            int32_t rc = (_e == cudaErrorMemoryAllocation) ? B200ADJ_ERR_OOM : B200ADJ_ERR_CUDA; \
            free_all(h); delete h; return rc; } } while (0)
        CREATE_TRY(cudaSetDevice(cfg->device));
        CREATE_TRY(cudaStreamCreateWithFlags(&h->own_stream, cudaStreamNonBlocking));
        h->stream = h->own_stream;
        const size_t N = (size_t)cfg->N, MS = (size_t)h->maxs, e = sizeof(double);
        if (t5a) {      // member-major records (u_n, k1..k7, t_n, h, 1/h, t_{n+1}) and knots: tsit5_adaptive.cuh
            CREATE_TRY(cudaMalloc(&h->r_ftT, N * (MS + 1) * e));
            CREATE_TRY(cudaMalloc(&h->r_frecT, N * (MS + 1) * (size_t)(8 * d + 4) * e));
        } else {
            CREATE_TRY(cudaMalloc(&h->r_ft, (MS + 1) * N * e));
            CREATE_TRY(cudaMalloc(&h->r_fu, (MS + 1) * d * N * e));
            CREATE_TRY(cudaMalloc(&h->r_fk, MS * h->nk * d * N * e));
        }
        CREATE_TRY(cudaMalloc(&h->r_fn, N * sizeof(int32_t)));
        CREATE_TRY(cudaMalloc(&h->r_rn, N * sizeof(int32_t)));
        h->maxseg = 2 * h->maxs;                                              // quadgk segment capacity per data interval (multiple of 32)
        {
            cudaDeviceGetAttribute(&h->nsm, cudaDevAttrMultiProcessorCount, cfg->device);
            h->qgrid = quad_grid(cfg->N, h->nsm);
        }
        CREATE_TRY(cudaMalloc(&h->d_saveat, (size_t)(cfg->K > 0 ? cfg->K : 1) * e));
        if (cfg->K > 0) CREATE_TRY(cudaMemcpy(h->d_saveat, cfg->saveat, (size_t)cfg->K * e, cudaMemcpyHostToDevice));
        // the forward pass keeps its own save table: set_reverse_options may re-target the reverse pass' jump times
        h->fwd_K = cfg->K; h->fwd_saveat = h->saveat;
        CREATE_TRY(cudaMalloc(&h->d_fwd_saveat, (size_t)(cfg->K > 0 ? cfg->K : 1) * e));
        if (cfg->K > 0) CREATE_TRY(cudaMemcpy(h->d_fwd_saveat, cfg->saveat, (size_t)cfg->K * e, cudaMemcpyHostToDevice));
        h->qpartials_blocks = (size_t)h->qgrid + 1;                              // quadrature kernel: persistent grid
        {   // block partials of the dG/dp reduction: the reverse kernels may run with blocks as small as one warp (disp_t5a.inc)
            const size_t gmax = (size_t)((cfg->N + 31) / 32);
            CREATE_TRY(cudaMalloc(&h->d_partials, (h->qpartials_blocks > gmax ? h->qpartials_blocks : gmax) * P * sizeof(double)));
        }
        CREATE_TRY(cudaMalloc(&h->d_ticket, sizeof(unsigned int)));
        CREATE_TRY(cudaMemset(h->d_ticket, 0, sizeof(unsigned int)));
        if (!cfg->buffers_on_device) {
            const size_t pn = cfg->shared_p ? (size_t)P : (size_t)P * N;
            CREATE_TRY(cudaMalloc(&h->s_u0, d * N * e));
            CREATE_TRY(cudaMalloc(&h->s_p, pn * e));
            CREATE_TRY(cudaMalloc(&h->s_du0, d * N * e));
            CREATE_TRY(cudaMalloc(&h->s_dp, pn * e));
            CREATE_TRY(cudaMalloc(&h->s_status, N * sizeof(int32_t)));
            if (cfg->K > 0) {
                CREATE_TRY(cudaMalloc(&h->s_saved, (size_t)cfg->K * d * N * e));
                if (cfg->cost_kind == B200ADJ_COST_EXPLICIT) CREATE_TRY(cudaMalloc(&h->s_dLdu, (size_t)cfg->K * d * N * e));
            }
        }
#undef CREATE_TRY
        for (int j = 0; j < 4; j++) { h->cost_av[j] = cfg->cost_a; h->cost_bv[j] = cfg->cost_b; }
        *handle = h;
        return B200ADJ_OK;
    }
    // fixed-step grid: the horizon must be a whole number of steps and every save time must be a grid point.
    // (Off-grid tstops split a step in the reference; that case is delegated back to the reference path.)
    const double span = cfg->t1 - cfg->t0;
    const double Sf = span / cfg->dt;
    const long long S = llround(Sf);
    if (S < 1 || S > 2000000000LL || fabs(S * cfg->dt - span) > 1e-9 * fmax(1.0, fabs(span))) {
        g_create_error = "(t1-t0) is not a whole number of dt steps"; return B200ADJ_ERR_UNSUPPORTED; }
    std::vector<int32_t> sos((size_t)S + 1, -1);
    for (int k = 0; k < cfg->K; k++) {
        const double tk = cfg->saveat[k];
        const long long n = llround((tk - cfg->t0) / cfg->dt);
        if (n < 0 || n > S || fabs(cfg->t0 + n * cfg->dt - tk) > 1e-9 * fmax(1.0, fabs(tk))) {
            g_create_error = "saveat entry is not on the dt grid"; return B200ADJ_ERR_UNSUPPORTED; }
        if (sos[n] != -1) { g_create_error = "duplicate save times are not supported"; return B200ADJ_ERR_UNSUPPORTED; }
        if (k > 0 && !(tk > cfg->saveat[k - 1])) { g_create_error = "saveat must be ascending"; return B200ADJ_ERR_INVALID; }
        sos[n] = k;
    }
    // Block size.  The reverse kernel is capped at 128 registers => at most 512 resident threads per SM; every thread
    // runs the whole time loop, so the grid must fit in whole waves.  Default: ONE block per SM (block-wide barriers
    // every few steps keep all warps of an SM in lockstep -- independent small blocks drift apart by >2x under the
    // highest-warp-id-first arbiter and the stragglers run the tail latency-bound), sized so that the blocks cover
    // the SMs evenly: block = ceil32(N / (nSM * waves)).
    int nsm = 132;
    cudaDeviceGetAttribute(&nsm, cudaDevAttrMultiProcessorCount, cfg->device);
    int block = cfg->block_threads;
    if (block == 0) {
        const long long waves = (cfg->N + (long long)nsm * 512 - 1) / ((long long)nsm * 512);
        long long per = (cfg->N + nsm * waves - 1) / (nsm * waves);
        block = (int)(((per + 31) / 32) * 32);
        if (block < 32) block = 32;
        if (block > 512) block = 512;
    }
    if (block < 32 || block > 512 || (block % 32) != 0) { g_create_error = "block_threads must be a multiple of 32 in [32, 512]"; return B200ADJ_ERR_INVALID; }
    if (mlp) block = MLP_TB;      // members per block (the kernels run MLP_THREADS threads per block)
    // interval checkpointing (a14): forward states every C steps, segments re-solved by the reverse kernel
    int ckpt_every = cfg->checkpoint_every > 1 ? cfg->checkpoint_every : 1;
    if (ckpt_every > 1) {
        if (mlp || sde || (cfg->sensealg != B200ADJ_SA_INTERPOLATING && cfg->sensealg != B200ADJ_SA_GAUSS)) {
            g_create_error = "checkpoint_every > 1: fixed-step Tsit5 with InterpolatingAdjoint / GaussAdjoint (the sensealgs that checkpoint in the reference)"; return B200ADJ_ERR_UNSUPPORTED; }
        if (ckpt_every > S) ckpt_every = (int)S;
        const size_t need = (size_t)ckpt_every * d * block * esz(*cfg);
        if (need > 160 * 1024) { g_create_error = "checkpoint_every * d * block_threads * sizeof(real) exceeds 160 KB of shared memory: lower checkpoint_every or block_threads"; return B200ADJ_ERR_INVALID; }
    }

    Handle* h = new Handle();
    h->cfg = *cfg; h->cfg.m = m;
    h->saveat.assign(cfg->saveat, cfg->saveat + cfg->K);
    h->cfg.saveat = h->saveat.data();
    h->save_of_step = sos;
    h->S = (int)S; h->block = block; h->ckpt_every = ckpt_every;
    h->grid = (int)((cfg->N + block - 1) / block);
#define CREATE_TRY(expr)                                                                         \
    do { cudaError_t _e = (expr); if (_e != cudaSuccess) {                                       \
        g_create_error = std::string(#expr) + ": " + cudaGetErrorString(_e);                     \
        int32_t rc = (_e == cudaErrorMemoryAllocation) ? B200ADJ_ERR_OOM : B200ADJ_ERR_CUDA;     \
        free_all(h); delete h; return rc; } } while (0)
    CREATE_TRY(cudaSetDevice(cfg->device));
    CREATE_TRY(cudaStreamCreateWithFlags(&h->own_stream, cudaStreamNonBlocking));
    h->stream = h->own_stream;
    const size_t N = (size_t)cfg->N, e = esz(*cfg);
    const size_t Npad = ((N + block - 1) / block) * block;     // padded checkpoint pitch (whole TMA rows per block)
    h->Npad = (int64_t)Npad;
    const size_t ckpt_rows = ckpt_every > 1 ? ((size_t)S + ckpt_every - 1) / ckpt_every + 1 : (size_t)S + 1;
    CREATE_TRY(cudaMalloc(&h->d_ckpt, ckpt_rows * d * Npad * e));
    h->nsm = nsm; h->qgrid = quad_grid(cfg->N, nsm);
    h->qpart_blocks_fixed = (size_t)h->qgrid + 1;
    CREATE_TRY(cudaMalloc(&h->d_partials, (h->qpart_blocks_fixed > (size_t)h->grid ? h->qpart_blocks_fixed : (size_t)h->grid) * P * sizeof(double)));
    CREATE_TRY(cudaMalloc(&h->d_ticket, sizeof(unsigned int)));
    CREATE_TRY(cudaMemset(h->d_ticket, 0, sizeof(unsigned int)));
    CREATE_TRY(cudaMalloc(&h->d_save_of_step, ((size_t)S + 1) * sizeof(int32_t)));
    CREATE_TRY(cudaMemcpy(h->d_save_of_step, sos.data(), ((size_t)S + 1) * sizeof(int32_t), cudaMemcpyHostToDevice));
    // the forward pass keeps its own save table: set_reverse_options may re-target the reverse pass' jump times
    h->fwd_K = cfg->K; h->fwd_saveat = h->saveat; h->fwd_save_of_step = sos;
    CREATE_TRY(cudaMalloc(&h->d_fwd_save_of_step, ((size_t)S + 1) * sizeof(int32_t)));
    CREATE_TRY(cudaMemcpy(h->d_fwd_save_of_step, sos.data(), ((size_t)S + 1) * sizeof(int32_t), cudaMemcpyHostToDevice));
    if (sde) CREATE_TRY(cudaMalloc(&h->d_noise, (size_t)S * m * N * e));
    // BF16_F32ACC = mlp_tc.cuh: member and gradient GEMMs in the time loop on wgmma, fp32 accumulators in registers
    h->mlp_tc = mlp && cfg->dtype == B200ADJ_BF16_F32ACC;
    if (h->mlp_tc) CREATE_TRY(cudaMalloc(&h->d_kst, (size_t)S * 14 * N * sizeof(float)));
    if (cfg->flags & B200ADJ_FLAG_TRACE) {
        CREATE_TRY(cudaMalloc(&h->d_trace, (size_t)h->grid * 3 * sizeof(unsigned long long)));
        CREATE_TRY(cudaMemset(h->d_trace, 0, (size_t)h->grid * 3 * sizeof(unsigned long long)));
    }
    if (!cfg->buffers_on_device) {
        const size_t pn = cfg->shared_p ? (size_t)P : (size_t)P * N;
        CREATE_TRY(cudaMalloc(&h->s_u0, d * N * e));
        CREATE_TRY(cudaMalloc(&h->s_p, pn * e));
        CREATE_TRY(cudaMalloc(&h->s_du0, d * N * e));
        CREATE_TRY(cudaMalloc(&h->s_dp, pn * e));
        CREATE_TRY(cudaMalloc(&h->s_status, N * sizeof(int32_t)));
        if (cfg->K > 0) {
            CREATE_TRY(cudaMalloc(&h->s_saved, (size_t)cfg->K * d * N * e));
            if (cfg->cost_kind == B200ADJ_COST_EXPLICIT) CREATE_TRY(cudaMalloc(&h->s_dLdu, (size_t)cfg->K * d * N * e));
        }
    }
#undef CREATE_TRY
    if (!sde) build_tsit5_tables(cfg->dt, &h->tb);
    for (int j = 0; j < 4; j++) { h->cost_av[j] = cfg->cost_a; h->cost_bv[j] = cfg->cost_b; }
    *handle = h;
    return B200ADJ_OK;
}

int32_t b200adj_set_reverse_options(void* handle, int32_t sensealg, int32_t cost_kind, double cost_a, double cost_b,
                                    uint32_t flags, int32_t K, const double* t) {
    if (!handle) return B200ADJ_ERR_INVALID;
    Handle* h = (Handle*)handle;
    b200adj_cfg& c = h->cfg;
    if (sensealg < 0 || sensealg > 4 || (cost_kind != B200ADJ_COST_EXPLICIT && cost_kind != B200ADJ_COST_AFFINE)) { h->err = "bad sensealg/cost_kind"; return B200ADJ_ERR_INVALID; }
    if (h->cc_on && sensealg == B200ADJ_SA_QUADRATURE) { h->err = "continuous callback: QuadratureAdjoint has no callback support"; return B200ADJ_ERR_UNSUPPORTED; }
    if (sensealg == B200ADJ_SA_GAUSSKRONROD && (is_sde(c) || c.rhs_family == B200ADJ_FAM_MLP || c.dtype != B200ADJ_F64)) { h->err = "GaussKronrodAdjoint: F64, named ODE families"; return B200ADJ_ERR_UNSUPPORTED; }
    if (h->ckpt_every > 1 && sensealg != B200ADJ_SA_INTERPOLATING && sensealg != B200ADJ_SA_GAUSS) { h->err = "checkpoint_every > 1: InterpolatingAdjoint / GaussAdjoint only"; return B200ADJ_ERR_UNSUPPORTED; }
    if (is_sde(c) && sensealg != B200ADJ_SA_BACKSOLVE && sensealg != B200ADJ_SA_INTERPOLATING) { h->err = "SDE: BacksolveAdjoint / InterpolatingAdjoint are built"; return B200ADJ_ERR_UNSUPPORTED; }
    if (c.rhs_family == B200ADJ_FAM_MLP && sensealg != B200ADJ_SA_INTERPOLATING && sensealg != B200ADJ_SA_GAUSS) { h->err = "MLP family: InterpolatingAdjoint / GaussAdjoint are built"; return B200ADJ_ERR_UNSUPPORTED; }
    if (h->nev > 0 && sensealg == B200ADJ_SA_QUADRATURE) { h->err = "events: QuadratureAdjoint has no callback support"; return B200ADJ_ERR_UNSUPPORTED; }
    if (c.dtype == B200ADJ_F32 && c.rhs_family != B200ADJ_FAM_MLP && sensealg == B200ADJ_SA_QUADRATURE) { h->err = "F32: QuadratureAdjoint is F64 only"; return B200ADJ_ERR_UNSUPPORTED; }
    CUDA_TRY(h, cudaSetDevice(c.device));
    if (h->adaptive) {
        if (K >= 0) {
            for (int k = 0; k < K; k++)
                if (t[k] < c.t0 || t[k] > c.t1 || (k > 0 && !(t[k] > t[k - 1]))) { h->err = "t must be ascending inside [t0, t1]"; return B200ADJ_ERR_INVALID; }
            CUDA_TRY(h, cudaStreamSynchronize(h->stream));
            if (K > c.K) { cudaFree(h->d_saveat); h->d_saveat = nullptr; CUDA_TRY(h, cudaMalloc(&h->d_saveat, (size_t)K * sizeof(double))); cudaFree(h->s_dLdu); h->s_dLdu = nullptr; }
            if (K > 0) CUDA_TRY(h, cudaMemcpy(h->d_saveat, t, (size_t)K * sizeof(double), cudaMemcpyHostToDevice));
            h->saveat.assign(t, t + K); c.saveat = h->saveat.data(); c.K = K;
        }
        if (!c.buffers_on_device && cost_kind == B200ADJ_COST_EXPLICIT && c.K > 0 && !h->s_dLdu)
            CUDA_TRY(h, cudaMalloc(&h->s_dLdu, (size_t)c.K * c.d * (size_t)c.N * esz(c)));
        c.sensealg = sensealg; c.cost_kind = cost_kind; c.cost_a = cost_a; c.cost_b = cost_b;
        for (int j = 0; j < 4; j++) { h->cost_av[j] = cost_a; h->cost_bv[j] = cost_b; }
        h->has_dgdp = false;
        c.flags = (c.flags & B200ADJ_CREATE_FLAGS) | (flags & ~B200ADJ_CREATE_FLAGS);
        return B200ADJ_OK;
    }
    if (K >= 0) {
        if (K > 0 && !t) { h->err = "null t"; return B200ADJ_ERR_INVALID; }
        std::vector<int32_t> sos((size_t)h->S + 1, -1);
        for (int k = 0; k < K; k++) {
            const long long n = llround((t[k] - c.t0) / c.dt);
            if (n < 0 || n > h->S || fabs(c.t0 + n * c.dt - t[k]) > 1e-9 * fmax(1.0, fabs(t[k]))) { h->err = "t entry is not on the dt grid"; return B200ADJ_ERR_UNSUPPORTED; }
            if (sos[n] != -1) { h->err = "duplicate save times are not supported"; return B200ADJ_ERR_UNSUPPORTED; }
            sos[n] = k;
        }
        CUDA_TRY(h, cudaStreamSynchronize(h->stream));
        CUDA_TRY(h, cudaMemcpy(h->d_save_of_step, sos.data(), sos.size() * sizeof(int32_t), cudaMemcpyHostToDevice));
        h->save_of_step = sos;
        h->saveat.assign(t, t + K);
        c.saveat = h->saveat.data();
        if (!c.buffers_on_device && K > c.K) {
            cudaFree(h->s_dLdu); h->s_dLdu = nullptr;
        }
        if (!c.buffers_on_device && cost_kind == B200ADJ_COST_EXPLICIT && K > 0 && !h->s_dLdu)
            CUDA_TRY(h, cudaMalloc(&h->s_dLdu, (size_t)K * c.d * (size_t)c.N * esz(c)));
        c.K = K;
    } else if (!c.buffers_on_device && cost_kind == B200ADJ_COST_EXPLICIT && c.K > 0 && !h->s_dLdu) {
        CUDA_TRY(h, cudaMalloc(&h->s_dLdu, (size_t)c.K * c.d * (size_t)c.N * esz(c)));
    }
    c.sensealg = sensealg; c.cost_kind = cost_kind; c.cost_a = cost_a; c.cost_b = cost_b;
    for (int j = 0; j < 4; j++) { h->cost_av[j] = cost_a; h->cost_bv[j] = cost_b; }
    h->has_dgdp = false;
    c.flags = (c.flags & B200ADJ_CREATE_FLAGS) | (flags & ~B200ADJ_CREATE_FLAGS);
    return B200ADJ_OK;
}

int32_t b200adj_set_continuous_cost(void* handle, int32_t enabled, double a, double b) {
    if (!handle) return B200ADJ_ERR_INVALID;
    Handle* h = (Handle*)handle;
    if (enabled && ((h->adaptive && h->cfg.stepper != B200ADJ_ST_TSIT5_ADAPTIVE && !h->fixed_dt) || is_sde(h->cfg) || h->cfg.rhs_family == B200ADJ_FAM_MLP)) {
        h->err = "continuous cost: built for the Tsit5 ODE paths (fixed step and adaptive)"; return B200ADJ_ERR_UNSUPPORTED; }
    h->cont_on = enabled != 0;
    for (int j = 0; j < 4; j++) { h->cont_av[j] = a; h->cont_bv[j] = b; }
    h->has_cdgdp = false;
    return B200ADJ_OK;
}

int32_t b200adj_register_family(const char* plugin_path, int32_t* family_id) {
    if (!plugin_path || !family_id) { g_create_error = "register_family: null argument"; return B200ADJ_ERR_INVALID; }
    void* lib = dlopen(plugin_path, RTLD_NOW | RTLD_LOCAL);
    if (!lib) { const char* e = dlerror(); g_create_error = std::string("register_family: dlopen failed: ") + (e ? e : "?"); return B200ADJ_ERR_INVALID; }
    typedef const FamilyVTable* (*entry_t)(void);
    entry_t entry = (entry_t)dlsym(lib, "b200adj_family_plugin");
    if (!entry) { dlclose(lib); g_create_error = "register_family: the library does not export b200adj_family_plugin"; return B200ADJ_ERR_INVALID; }
    const FamilyVTable* vt = entry();
    // a refused plug-in is unloaded again, so that a rebuilt file of the same name is really loaded next time
    if (!vt || vt->abi != B200ADJ_PLUGIN_ABI) { dlclose(lib); g_create_error = "register_family: plug-in built against other headers (ABI tag mismatch): rebuild it"; return B200ADJ_ERR_INVALID; }
    if (vt->d < 1 || vt->d > 4 || vt->P < 1 || vt->P > 8) { dlclose(lib); g_create_error = "register_family: 1 <= D <= 4 and 1 <= P <= 8"; return B200ADJ_ERR_UNSUPPORTED; }
    auto& r = family_registry();
    for (size_t k = 0; k < r.size(); k++) if (r[k] == vt) { *family_id = B200ADJ_FAM_USER_BASE_ID + (int)k; return B200ADJ_OK; }
    r.push_back(vt);
    *family_id = B200ADJ_FAM_USER_BASE_ID + (int)r.size() - 1;
    return B200ADJ_OK;
}

int32_t b200adj_family_info(int32_t family_id, int32_t* d, int32_t* P, const char** name) {
    const FamilyVTable* vt = family_lookup(family_id);
    if (!vt) return B200ADJ_ERR_INVALID;
    if (d) *d = vt->d;
    if (P) *P = vt->P;
    if (name) *name = vt->name;
    return B200ADJ_OK;
}

int32_t b200adj_set_cost_family(void* handle, int32_t which, const double* a, const double* b, const double* c, const double* e) {
    if (!handle || (which != 0 && which != 1)) return B200ADJ_ERR_INVALID;
    Handle* h = (Handle*)handle;
    const b200adj_cfg& cf = h->cfg;
    if ((c || e) && (cf.P > 8 || cf.rhs_family == B200ADJ_FAM_MLP)) { h->err = "cost family: the parameter part (dgdp) is built for P <= 8"; return B200ADJ_ERR_UNSUPPORTED; }
    if ((c || e) && h->d_ev_ps) { h->err = "cost family: dgdp together with parameter-changing events is not built"; return B200ADJ_ERR_UNSUPPORTED; }
    if (which == 1) {
        int32_t rc = b200adj_set_continuous_cost(handle, 1, 0.0, 0.0);       // same support matrix as the scalar entry point
        if (rc) return rc;
    } else if (cf.cost_kind != B200ADJ_COST_AFFINE && (a || b)) { h->err = "cost family: per-component dgdu_discrete needs cost_kind = AFFINE"; return B200ADJ_ERR_INVALID; }
    double* av = which ? h->cont_av : h->cost_av; double* bv = which ? h->cont_bv : h->cost_bv;
    double* cv = which ? h->cdgdp_c : h->dgdp_c; double* ev = which ? h->cdgdp_e : h->dgdp_e;
    for (int j = 0; j < 4; j++) { if (a) av[j] = j < cf.d ? a[j] : 0.0; if (b) bv[j] = j < cf.d ? b[j] : 0.0; }
    for (int q = 0; q < 8; q++) { cv[q] = (c && q < cf.P) ? c[q] : 0.0; ev[q] = (e && q < cf.P) ? e[q] : 0.0; }
    (which ? h->has_cdgdp : h->has_dgdp) = (c != nullptr || e != nullptr);
    return B200ADJ_OK;
}

int32_t b200adj_set_events(void* handle, int32_t E, const double* times, const double* scale, const double* shift,
                           const double* pscale, const double* pshift) {
    if (!handle) return B200ADJ_ERR_INVALID;
    Handle* h = (Handle*)handle;
    const b200adj_cfg& c = h->cfg;
    if (E < 0 || (E > 0 && (!times || !scale || !shift)) || ((pscale == nullptr) != (pshift == nullptr))) { h->err = "set_events: bad arguments"; return B200ADJ_ERR_INVALID; }
    if (E > 0 && h->cc_on) { h->err = "events: preset-time events together with a continuous callback are not built"; return B200ADJ_ERR_UNSUPPORTED; }
    // hybrid neural ODE (test/Core5/HybridNODE.jl): the MLP family's CUDA-core kernels (F64 / F32) carry state events on the dt grid
    const bool mlp_ev = c.rhs_family == B200ADJ_FAM_MLP && !h->mlp_tc && c.stepper == B200ADJ_ST_TSIT5_FIXED;
    const bool fixed = c.stepper == B200ADJ_ST_TSIT5_FIXED && !h->fixed_dt && ((c.rhs_family != B200ADJ_FAM_MLP && c.dtype == B200ADJ_F64) || mlp_ev);
    if (E > 0 && c.stepper != B200ADJ_ST_TSIT5_ADAPTIVE && !fixed && !h->fixed_dt) { h->err = "events: built for the Tsit5 steppers (adaptive; fixed step in F64; MLP family: F64 / F32, not the bf16 tensor-core path)"; return B200ADJ_ERR_UNSUPPORTED; }
    if (E > 0 && mlp_ev && pscale) { h->err = "events: parameter-changing affects are not built for the MLP family"; return B200ADJ_ERR_UNSUPPORTED; }
    if (E > 0 && fixed && h->ckpt_every > 1) { h->err = "events together with checkpoint_every > 1 are not built"; return B200ADJ_ERR_UNSUPPORTED; }
    std::vector<int32_t> eos;
    if (fixed) {
        // fixed step: every event time must be a grid point (the affect is applied between two steps)
        eos.assign((size_t)h->S + 1, -1);
        for (int e = 0; e < E; e++) {
            const long long n = llround((times[e] - c.t0) / c.dt);
            if (n <= 0 || n >= h->S || fabs(c.t0 + n * c.dt - times[e]) > 1e-9 * fmax(1.0, fabs(times[e]))) { h->err = "events: fixed-step Tsit5 needs event times on the dt grid, strictly inside (t0, t1)"; return B200ADJ_ERR_UNSUPPORTED; }
            if (eos[n] != -1) { h->err = "events: duplicate event times"; return B200ADJ_ERR_INVALID; }
            eos[n] = e;
        }
    }
    if (E > 0 && c.sensealg == B200ADJ_SA_QUADRATURE) { h->err = "events: Interpolating / Gauss / Backsolve (QuadratureAdjoint has no callback support)"; return B200ADJ_ERR_UNSUPPORTED; }
    for (int e = 0; e < E; e++)
        if (!(times[e] > c.t0 && times[e] < c.t1) || (e > 0 && !(times[e] > times[e - 1]))) { h->err = "events: times must be ascending and strictly inside (t0, t1)"; return B200ADJ_ERR_INVALID; }
    CUDA_TRY(h, cudaSetDevice(c.device));
    CUDA_TRY(h, cudaStreamSynchronize(h->stream));
    cudaFree(h->d_ev_t); cudaFree(h->d_ev_s); cudaFree(h->d_ev_c); cudaFree(h->d_ev_ps); cudaFree(h->d_ev_pc);
    cudaFree(h->d_ev_ac); cudaFree(h->d_ev_ak); cudaFree(h->d_ev_af); h->d_ev_ac = h->d_ev_ak = nullptr; h->d_ev_af = nullptr;
    h->d_ev_t = h->d_ev_s = h->d_ev_c = h->d_ev_ps = h->d_ev_pc = nullptr; h->nev = 0; h->have_forward = false;
    if (E > 0) {
        CUDA_TRY(h, cudaMalloc(&h->d_ev_t, (size_t)E * sizeof(double)));
        CUDA_TRY(h, cudaMalloc(&h->d_ev_s, (size_t)E * c.d * sizeof(double)));
        CUDA_TRY(h, cudaMalloc(&h->d_ev_c, (size_t)E * c.d * sizeof(double)));
        CUDA_TRY(h, cudaMemcpy(h->d_ev_t, times, (size_t)E * sizeof(double), cudaMemcpyHostToDevice));
        CUDA_TRY(h, cudaMemcpy(h->d_ev_s, scale, (size_t)E * c.d * sizeof(double), cudaMemcpyHostToDevice));
        CUDA_TRY(h, cudaMemcpy(h->d_ev_c, shift, (size_t)E * c.d * sizeof(double), cudaMemcpyHostToDevice));
        if (pscale) {
            CUDA_TRY(h, cudaMalloc(&h->d_ev_ps, (size_t)E * c.P * sizeof(double)));
            CUDA_TRY(h, cudaMalloc(&h->d_ev_pc, (size_t)E * c.P * sizeof(double)));
            CUDA_TRY(h, cudaMemcpy(h->d_ev_ps, pscale, (size_t)E * c.P * sizeof(double), cudaMemcpyHostToDevice));
            CUDA_TRY(h, cudaMemcpy(h->d_ev_pc, pshift, (size_t)E * c.P * sizeof(double), cudaMemcpyHostToDevice));
        }
        h->nev = E;
    }
    if (fixed) {
        if (!h->d_event_of_step) CUDA_TRY(h, cudaMalloc(&h->d_event_of_step, ((size_t)h->S + 1) * sizeof(int32_t)));
        CUDA_TRY(h, cudaMemcpy(h->d_event_of_step, eos.data(), eos.size() * sizeof(int32_t), cudaMemcpyHostToDevice));
    }
    return B200ADJ_OK;
}

int32_t b200adj_set_event_param_shift(void* handle, const int32_t* comp, const int32_t* param, const double* coef) {
    if (!handle) return B200ADJ_ERR_INVALID;
    Handle* h = (Handle*)handle;
    const b200adj_cfg& c = h->cfg;
    if (h->nev <= 0) { h->err = "event parameter shift: call b200adj_set_events first"; return B200ADJ_ERR_STATE; }
    CUDA_TRY(h, cudaSetDevice(c.device));
    CUDA_TRY(h, cudaStreamSynchronize(h->stream));
    cudaFree(h->d_ev_ac); cudaFree(h->d_ev_ak); cudaFree(h->d_ev_af); h->d_ev_ac = h->d_ev_ak = nullptr; h->d_ev_af = nullptr;
    h->have_forward = false;
    if (!comp) return B200ADJ_OK;                                      // removes the shifts
    if (!param || !coef) { h->err = "event parameter shift: null argument"; return B200ADJ_ERR_INVALID; }
    if (!(c.stepper == B200ADJ_ST_TSIT5_ADAPTIVE || h->fixed_dt)) {
        h->err = "event parameter shift: built on the per-member dense framework (adaptive Tsit5, or fixed step with B200ADJ_FLAG_DENSE_FORWARD)";
        return B200ADJ_ERR_UNSUPPORTED; }
    for (int e = 0; e < h->nev; e++)
        if (comp[e] >= c.d || (comp[e] >= 0 && (param[e] < 0 || param[e] >= c.P || !std::isfinite(coef[e])))) {
            h->err = "event parameter shift: bad component / parameter index"; return B200ADJ_ERR_INVALID; }
    const size_t E = (size_t)h->nev;
    CUDA_TRY(h, cudaMalloc(&h->d_ev_ac, E * sizeof(int32_t)));
    CUDA_TRY(h, cudaMalloc(&h->d_ev_ak, E * sizeof(int32_t)));
    CUDA_TRY(h, cudaMalloc(&h->d_ev_af, E * sizeof(double)));
    CUDA_TRY(h, cudaMemcpy(h->d_ev_ac, comp, E * sizeof(int32_t), cudaMemcpyHostToDevice));
    CUDA_TRY(h, cudaMemcpy(h->d_ev_ak, param, E * sizeof(int32_t), cudaMemcpyHostToDevice));
    CUDA_TRY(h, cudaMemcpy(h->d_ev_af, coef, E * sizeof(double), cudaMemcpyHostToDevice));
    return B200ADJ_OK;
}

int32_t b200adj_set_continuous_callback(void* handle, int32_t enabled, int32_t idx, double level, int32_t direction,
                                        const double* scale, const double* shift, int32_t pcomp, int32_t pparam, double psign,
                                        int32_t max_events) {
    if (!handle) return B200ADJ_ERR_INVALID;
    Handle* h = (Handle*)handle;
    const b200adj_cfg& c = h->cfg;
    CUDA_TRY(h, cudaSetDevice(c.device));
    CUDA_TRY(h, cudaStreamSynchronize(h->stream));
    if (!enabled) {
        cudaFree(h->d_cc_t); cudaFree(h->d_cc_n); h->d_cc_t = nullptr; h->d_cc_n = nullptr; h->cc_on = false; h->have_forward = false;
        return B200ADJ_OK;
    }
    if (c.stepper != B200ADJ_ST_TSIT5_ADAPTIVE || h->fixed_dt || c.dtype != B200ADJ_F64) { h->err = "continuous callback: built for the adaptive Tsit5 stepper (F64)"; return B200ADJ_ERR_UNSUPPORTED; }
    if (c.sensealg == B200ADJ_SA_QUADRATURE) { h->err = "continuous callback: Interpolating / Gauss / GaussKronrod / Backsolve (QuadratureAdjoint has no callback support)"; return B200ADJ_ERR_UNSUPPORTED; }
    if (h->nev > 0) { h->err = "continuous callback together with preset-time events is not built"; return B200ADJ_ERR_UNSUPPORTED; }
    if (c.d > 4) { h->err = "continuous callback: d <= 4"; return B200ADJ_ERR_UNSUPPORTED; }
    if (idx < 0 || idx >= c.d || direction < -1 || direction > 1 || pcomp >= c.d || (pcomp >= 0 && (pparam < 0 || pparam >= c.P)) || max_events < 1 ||
        !std::isfinite(level) || !std::isfinite(psign)) { h->err = "continuous callback: bad idx / direction / pcomp / pparam / max_events"; return B200ADJ_ERR_INVALID; }
    if ((size_t)max_events != (size_t)h->cc_maxev || !h->d_cc_t) {
        cudaFree(h->d_cc_t); cudaFree(h->d_cc_n); h->d_cc_t = nullptr; h->d_cc_n = nullptr; h->cc_on = false;
        CUDA_TRY(h, cudaMalloc(&h->d_cc_t, (size_t)max_events * (size_t)c.N * sizeof(double)));
        CUDA_TRY(h, cudaMalloc(&h->d_cc_n, (size_t)c.N * sizeof(int32_t)));
    }
    CUDA_TRY(h, cudaMemsetAsync(h->d_cc_n, 0, (size_t)c.N * sizeof(int32_t), h->stream));
    h->cc_on = true; h->cc_idx = idx; h->cc_dir = direction; h->cc_pcomp = pcomp < 0 ? -1 : pcomp; h->cc_pparam = pcomp < 0 ? 0 : pparam;
    h->cc_maxev = max_events; h->cc_level = level; h->cc_psign = psign;
    h->cc_lparam = -1; h->cc_lcoef = 0; h->cc_acomp = -1; h->cc_aparam = 0; h->cc_acoef = 0; h->cc_qcomp = -1; h->cc_qcoef = 1;   // set_continuous_callback_params adds them
    for (int j = 0; j < 4; j++) { h->cc_scale[j] = (scale && j < c.d) ? scale[j] : 1.0; h->cc_shift[j] = (shift && j < c.d) ? shift[j] : 0.0; }
    h->have_forward = false;
    return B200ADJ_OK;
}

int32_t b200adj_set_continuous_callback_params(void* handle, int32_t lparam, double lcoef, int32_t acomp, int32_t aparam, double acoef,
                                               int32_t qcomp, double qcoef) {
    if (!handle) return B200ADJ_ERR_INVALID;
    Handle* h = (Handle*)handle;
    const b200adj_cfg& c = h->cfg;
    if (!h->cc_on) { h->err = "continuous callback parameters: call b200adj_set_continuous_callback first"; return B200ADJ_ERR_STATE; }
    if (lparam >= c.P || (acomp >= 0 && (acomp >= c.d || aparam < 0 || aparam >= c.P)) || !std::isfinite(lcoef) || !std::isfinite(acoef)) {
        h->err = "continuous callback parameters: bad lparam / acomp / aparam"; return B200ADJ_ERR_INVALID; }
    if (acomp >= 0 && acomp == h->cc_pcomp) { h->err = "continuous callback parameters: acomp is the component the parameter-scaled affect overwrites"; return B200ADJ_ERR_INVALID; }
    if (qcomp >= c.d || !std::isfinite(qcoef) || (qcomp >= 0 && (qcomp == h->cc_pcomp || qcomp == acomp))) {
        h->err = "continuous callback parameters: bad qcomp (a component no other part of the affect writes)"; return B200ADJ_ERR_INVALID; }
    CUDA_TRY(h, cudaSetDevice(c.device));
    CUDA_TRY(h, cudaStreamSynchronize(h->stream));
    h->cc_lparam = lparam < 0 ? -1 : lparam; h->cc_lcoef = lparam < 0 ? 0.0 : lcoef;
    h->cc_acomp = acomp < 0 ? -1 : acomp; h->cc_aparam = acomp < 0 ? 0 : aparam; h->cc_acoef = acomp < 0 ? 0.0 : acoef;
    h->cc_qcomp = qcomp < 0 ? -1 : qcomp; h->cc_qcoef = qcomp < 0 ? 1.0 : qcoef;
    h->have_forward = false;
    return B200ADJ_OK;
}

int32_t b200adj_event_times(void* handle, int32_t* counts, double* times) {
    if (!handle) return B200ADJ_ERR_INVALID;
    Handle* h = (Handle*)handle;
    if (!h->cc_on || !h->have_forward) { h->err = "event_times: needs a continuous callback and a forward pass"; return B200ADJ_ERR_STATE; }
    CUDA_TRY(h, cudaSetDevice(h->cfg.device));
    CUDA_TRY(h, cudaStreamSynchronize(h->stream));
    if (counts) CUDA_TRY(h, cudaMemcpy(counts, h->d_cc_n, (size_t)h->cfg.N * sizeof(int32_t), cudaMemcpyDeviceToHost));
    if (times) CUDA_TRY(h, cudaMemcpy(times, h->d_cc_t, (size_t)h->cc_maxev * (size_t)h->cfg.N * sizeof(double), cudaMemcpyDeviceToHost));
    return B200ADJ_OK;
}

int32_t b200adj_set_tolerances(void* handle, double adj_abstol, double adj_reltol, double quad_abstol, double quad_reltol) {
    if (!handle) return B200ADJ_ERR_INVALID;
    Handle* h = (Handle*)handle;
    if (adj_abstol > 0) h->adj_abstol = adj_abstol;
    if (adj_reltol > 0) h->adj_reltol = adj_reltol;
    if (quad_abstol > 0) h->cfg.quad_abstol = quad_abstol;
    if (quad_reltol > 0) h->cfg.quad_reltol = quad_reltol;
    return B200ADJ_OK;
}

int32_t b200adj_set_stream(void* handle, void* cuda_stream) {
    if (!handle) return B200ADJ_ERR_INVALID;
    Handle* h = (Handle*)handle;
    h->stream = cuda_stream ? (cudaStream_t)cuda_stream : h->own_stream;
    return B200ADJ_OK;
}

int32_t b200adj_synchronize(void* handle) {
    if (!handle) return B200ADJ_ERR_INVALID;
    Handle* h = (Handle*)handle;
    CUDA_TRY(h, cudaSetDevice(h->cfg.device));
    CUDA_TRY(h, cudaStreamSynchronize(h->stream));
    return B200ADJ_OK;
}

int64_t b200adj_launch_count(void* handle) { return handle ? ((Handle*)handle)->launches : -1; }

int32_t b200adj_get_step_counts(void* handle, int32_t* fwd_steps, int32_t* rev_steps) {
    if (!handle) return B200ADJ_ERR_INVALID;
    Handle* h = (Handle*)handle;
    if (!h->adaptive) { h->err = "fixed-step handle: step count is S for every member"; return B200ADJ_ERR_UNSUPPORTED; }
    CUDA_TRY(h, cudaSetDevice(h->cfg.device));
    const cudaMemcpyKind kind = h->cfg.buffers_on_device ? cudaMemcpyDeviceToDevice : cudaMemcpyDeviceToHost;
    if (fwd_steps) CUDA_TRY(h, cudaMemcpyAsync(fwd_steps, h->r_fn, (size_t)h->cfg.N * sizeof(int32_t), kind, h->stream));
    if (rev_steps) CUDA_TRY(h, cudaMemcpyAsync(rev_steps, h->r_rn, (size_t)h->cfg.N * sizeof(int32_t), kind, h->stream));
    CUDA_TRY(h, cudaStreamSynchronize(h->stream));
    return B200ADJ_OK;
}

int32_t b200adj_forward(void* handle, const void* u0, const void* p, const void* dW_in, void* saved, int32_t* status) {
    if (!handle) return B200ADJ_ERR_INVALID;
    Handle* h = (Handle*)handle;
    const b200adj_cfg& c = h->cfg;
    if (!u0 || !p) { h->err = "null u0/p"; return B200ADJ_ERR_INVALID; }
    CUDA_TRY(h, cudaSetDevice(c.device));
    const size_t N = (size_t)c.N, e = esz(c);
    const size_t pn = c.shared_p ? (size_t)c.P : (size_t)c.P * N;
    const double *du0 = (const double*)u0, *dp = (const double*)p;
    double* dsaved = (double*)saved;
    int32_t* dstatus = status;
    if (!c.buffers_on_device) {
        CUDA_TRY(h, cudaMemcpyAsync(h->s_u0, u0, c.d * N * e, cudaMemcpyHostToDevice, h->stream));
        CUDA_TRY(h, cudaMemcpyAsync(h->s_p, p, pn * e, cudaMemcpyHostToDevice, h->stream));
        du0 = h->s_u0; dp = h->s_p;
        dsaved = (saved && h->fwd_K > 0) ? h->s_saved : nullptr;
        dstatus = status ? h->s_status : nullptr;
    }
    h->cur_p = dp;
    int rc = 0;
    if (h->adaptive && (c.stepper == B200ADJ_ST_TSIT5_ADAPTIVE || h->fixed_dt)) {
        T5aArgs a = t5a_args(h);
        a.saveat = h->d_fwd_saveat; a.K = h->fwd_K;
        a.u0 = du0; a.p = dp; a.saved = h->fwd_K > 0 ? dsaved : nullptr; a.status = dstatus;
        switch (c.rhs_family) {
        case B200ADJ_FAM_LV: rc = launch_t5a_fwd<LotkaVolterra>(h, a); break;
        case B200ADJ_FAM_LORENZ: rc = launch_t5a_fwd<Lorenz>(h, a); break;
        case B200ADJ_FAM_ROBERTSON: rc = launch_t5a_fwd<Robertson>(h, a); break;
        case B200ADJ_FAM_BALL: rc = launch_t5a_fwd<BouncingBall>(h, a); break;
        case B200ADJ_FAM_RELAX: rc = launch_t5a_fwd<Relax>(h, a); break;
        default: { const FamilyVTable* vt = family_lookup(c.rhs_family); rc = (vt && vt->t5a_fwd) ? vt->t5a_fwd(h, a) : B200ADJ_ERR_UNSUPPORTED; }
        }
    } else if (h->adaptive) {
        RosArgs a = ros_args(h);
        a.saveat = h->d_fwd_saveat; a.K = h->fwd_K;
        a.u0 = du0; a.p = dp; a.saved = h->fwd_K > 0 ? dsaved : nullptr; a.status = dstatus;
        switch (c.rhs_family) {
        case B200ADJ_FAM_LV: rc = launch_ros_fwd<LotkaVolterra>(h, a); break;
        case B200ADJ_FAM_LORENZ: rc = launch_ros_fwd<Lorenz>(h, a); break;
        case B200ADJ_FAM_ROBERTSON: rc = launch_ros_fwd<Robertson>(h, a); break;
        default: { const FamilyVTable* vt = family_lookup(c.rhs_family); rc = (vt && vt->ros_fwd) ? vt->ros_fwd(h, a) : B200ADJ_ERR_UNSUPPORTED; }
        }
    } else if (c.rhs_family == B200ADJ_FAM_MLP) {
        rc = mlp_forward_dispatch(h, du0, dp, h->fwd_K > 0 ? dsaved : nullptr, dstatus);
    } else if (!is_sde(c) && c.dtype == B200ADJ_F32) {
        OdeFwdArgsT<float> a;
        memset(&a, 0, sizeof(a));
        a.u0 = (const float*)du0; a.p = (const float*)dp; a.ckpt = (float*)h->d_ckpt; a.saved = h->fwd_K > 0 ? (float*)dsaved : nullptr;
        a.save_of_step = h->d_fwd_save_of_step; a.status = dstatus; a.N = c.N; a.Npad = h->Npad; a.S = h->S; a.ckpt_every = h->ckpt_every;
        cast_tables(h->tb, &a.tb);
        switch (c.rhs_family) {
        case B200ADJ_FAM_LV: rc = launch_fwd_f32<LotkaVolterra>(h, a); break;
        case B200ADJ_FAM_LORENZ: rc = launch_fwd_f32<Lorenz>(h, a); break;
        default: rc = B200ADJ_ERR_UNSUPPORTED;
        }
    } else if (!is_sde(c)) {
        OdeFwdArgs a;
        memset(&a, 0, sizeof(a));
        a.u0 = du0; a.p = dp; a.ckpt = h->d_ckpt; a.saved = h->fwd_K > 0 ? dsaved : nullptr; a.save_of_step = h->d_fwd_save_of_step;
        a.status = dstatus; a.N = c.N; a.Npad = h->Npad; a.S = h->S; a.tb = h->tb; a.ckpt_every = h->ckpt_every;
        a.event_of_step = h->d_event_of_step; a.ev_s = h->d_ev_s; a.ev_c = h->d_ev_c; a.ev_ps = h->d_ev_ps; a.ev_pc = h->d_ev_pc; a.nev = h->nev;
        switch (c.rhs_family) {
        case B200ADJ_FAM_LV: rc = launch_fwd<LotkaVolterra>(h, a); break;
        case B200ADJ_FAM_LORENZ: rc = launch_fwd<Lorenz>(h, a); break;
        case B200ADJ_FAM_ROBERTSON: rc = launch_fwd<Robertson>(h, a); break;
        default: { const FamilyVTable* vt = family_lookup(c.rhs_family); rc = (vt && vt->fwd) ? vt->fwd(h, a) : B200ADJ_ERR_UNSUPPORTED; }
        }
    } else {
        SdeFwdArgs a;
        a.u0 = du0; a.p = dp; a.ckpt = h->d_ckpt; a.saved = h->fwd_K > 0 ? dsaved : nullptr; a.save_of_step = h->d_fwd_save_of_step;
        a.status = dstatus; a.N = c.N; a.S = h->S; a.h = c.dt; a.seed = c.seed; a.traj_offset = c.traj_offset;
        // noise: (1) caller-supplied increments (parity tests, reference-style NoiseGrid) are copied into the handle;
        // (2) STORED_NOISE: Philox increments are written out by the forward kernel; (3) default: Philox, regenerated
        // by the reverse kernel (no HBM traffic for the noise).
        a.noise_in = nullptr; a.noise_out = nullptr;
        if (dW_in) {
            CUDA_TRY(h, cudaMemcpyAsync(h->d_noise, dW_in, (size_t)h->S * c.m * N * e,
                                        c.buffers_on_device ? cudaMemcpyDeviceToDevice : cudaMemcpyHostToDevice, h->stream));
            a.noise_in = h->d_noise; h->noise_valid = true;
        } else if (c.flags & B200ADJ_FLAG_STORED_NOISE) {
            a.noise_out = h->d_noise; h->noise_valid = true;
        } else {
            h->noise_valid = false;
        }
        rc = sde_forward_dispatch(h, a);
    }
    if (rc) { h->err = "forward dispatch failed"; return rc; }
    CUDA_TRY(h, cudaGetLastError());
    if (!c.buffers_on_device) {
        if (saved && h->fwd_K > 0) CUDA_TRY(h, cudaMemcpyAsync(saved, h->s_saved, (size_t)h->fwd_K * c.d * N * e, cudaMemcpyDeviceToHost, h->stream));
        if (status) CUDA_TRY(h, cudaMemcpyAsync(status, h->s_status, N * sizeof(int32_t), cudaMemcpyDeviceToHost, h->stream));
        CUDA_TRY(h, cudaStreamSynchronize(h->stream));
    }
    h->have_forward = true;
    return B200ADJ_OK;
}

int32_t b200adj_reverse(void* handle, const void* dLdu, void* du0, void* dp) {
    if (!handle) return B200ADJ_ERR_INVALID;
    Handle* h = (Handle*)handle;
    const b200adj_cfg& c = h->cfg;
    if (!h->have_forward) { h->err = "reverse called before forward"; return B200ADJ_ERR_STATE; }
    if (!du0 || !dp) { h->err = "null du0/dp"; return B200ADJ_ERR_INVALID; }
    if (c.cost_kind == B200ADJ_COST_EXPLICIT && c.K > 0 && !dLdu) { h->err = "COST_EXPLICIT needs dLdu"; return B200ADJ_ERR_INVALID; }
    CUDA_TRY(h, cudaSetDevice(c.device));
    const size_t N = (size_t)c.N, e = esz(c);
    const size_t pn = c.shared_p ? (size_t)c.P : (size_t)c.P * N;
    const double* dL = (const double*)dLdu;
    double *ddu0 = (double*)du0, *ddp = (double*)dp;
    if (!c.buffers_on_device) {
        if (c.cost_kind == B200ADJ_COST_EXPLICIT && c.K > 0) {
            CUDA_TRY(h, cudaMemcpyAsync(h->s_dLdu, dLdu, (size_t)c.K * c.d * N * e, cudaMemcpyHostToDevice, h->stream));
            dL = h->s_dLdu;
        }
        ddu0 = h->s_du0; ddp = h->s_dp;
    }
    int rc = 0;
    bool fused_allreduce = false;
    if (h->adaptive && (c.stepper == B200ADJ_ST_TSIT5_ADAPTIVE || h->fixed_dt)) {
        T5aArgs a = t5a_args(h);
        a.p = h->cur_p; a.dLdu = dL; a.du0 = ddu0; a.dp_members = ddp; a.dp = ddp;
        if (h->adj_abstol > 0) a.abstol = h->adj_abstol;
        if (h->adj_reltol > 0) a.reltol = h->adj_reltol;
        switch (c.rhs_family) {
        case B200ADJ_FAM_LV: rc = launch_t5a_rev<LotkaVolterra>(h, a); break;
        case B200ADJ_FAM_LORENZ: rc = launch_t5a_rev<Lorenz>(h, a); break;
        case B200ADJ_FAM_ROBERTSON: rc = launch_t5a_rev<Robertson>(h, a); break;
        case B200ADJ_FAM_BALL: rc = launch_t5a_rev<BouncingBall>(h, a); break;
        case B200ADJ_FAM_RELAX: rc = launch_t5a_rev<Relax>(h, a); break;
        default: { const FamilyVTable* vt = family_lookup(c.rhs_family); rc = (vt && vt->t5a_rev) ? vt->t5a_rev(h, a) : B200ADJ_ERR_UNSUPPORTED; }
        }
    } else if (h->adaptive) {
        RosArgs a = ros_args(h);
        a.p = h->cur_p; a.dLdu = dL; a.du0 = ddu0; a.dp_members = ddp; a.dp = ddp;
        if (h->adj_abstol > 0) a.abstol = h->adj_abstol;
        if (h->adj_reltol > 0) a.reltol = h->adj_reltol;
        switch (c.rhs_family) {
        case B200ADJ_FAM_LV: rc = launch_ros_rev<LotkaVolterra>(h, a); break;
        case B200ADJ_FAM_LORENZ: rc = launch_ros_rev<Lorenz>(h, a); break;
        case B200ADJ_FAM_ROBERTSON: rc = launch_ros_rev<Robertson>(h, a); break;
        default: { const FamilyVTable* vt = family_lookup(c.rhs_family); rc = (vt && vt->ros_rev) ? vt->ros_rev(h, a) : B200ADJ_ERR_UNSUPPORTED; }
        }
    } else if (c.rhs_family == B200ADJ_FAM_MLP) {
        rc = mlp_reverse_dispatch(h, dL, ddu0, ddp);
    } else if (!is_sde(c) && c.dtype == B200ADJ_F32) {
        if (h->cont_on) { h->err = "continuous cost: F64 only"; return B200ADJ_ERR_UNSUPPORTED; }
        OdeRevArgsT<float> a;
        memset(&a, 0, sizeof(a));
        a.ckpt = (const float*)h->d_ckpt; a.p = (const float*)h->cur_p; a.dLdu = (const float*)dL; a.save_of_step = h->d_save_of_step;
        a.du0 = (float*)ddu0; a.dp_members = (float*)ddp; a.partials = h->d_partials; a.dp = (float*)ddp; a.ticket = h->d_ticket;
        a.N = c.N; a.Npad = h->Npad; a.S = h->S; a.trace = h->d_trace;
        for (int j = 0; j < 4; j++) { a.cost_a[j] = (float)h->cost_av[j]; a.cost_b[j] = (float)h->cost_bv[j]; }
        cast_tables(h->tb, &a.tb);
        a.flags = ((c.flags & B200ADJ_FLAG_NO_START) ? 1u : 0u) | ((c.flags & B200ADJ_FLAG_NO_CHECKPOINTING) ? 2u : 0u) |
                  ((c.flags & B200ADJ_FLAG_CKPT_EVERY_STEP) ? 4u : 0u);
        switch (c.rhs_family) {
        case B200ADJ_FAM_LV: rc = launch_rev_f32<LotkaVolterra>(h, a); break;
        case B200ADJ_FAM_LORENZ: rc = launch_rev_f32<Lorenz>(h, a); break;
        default: rc = B200ADJ_ERR_UNSUPPORTED;
        }
    } else if (!is_sde(c)) {
        OdeRevArgs a;
        memset(&a, 0, sizeof(a));
        a.event_of_step = h->d_event_of_step; a.ev_s = h->d_ev_s; a.ev_c = h->d_ev_c; a.ev_ps = h->d_ev_ps; a.ev_pc = h->d_ev_pc; a.nev = h->nev;
        tsit5_weights(0.0, nullptr, a.Rpoly); a.hstep = c.dt;
        if (c.shared_p && comm_fused_ready(h) && !(c.flags & B200ADJ_FLAG_NCCL_ALLREDUCE) && c.sensealg != B200ADJ_SA_QUADRATURE && !h->has_dgdp && !(h->has_cdgdp && h->cont_on)) {
            // the all-reduce of dp is fused into this kernel's last block (peer-memory mailboxes): no collective launch
            a.p2p = h->p2p; a.p2p.epoch = ++h->p2p_epoch; fused_allreduce = true;
        }
        a.ckpt = h->d_ckpt; a.p = h->cur_p; a.dLdu = dL; a.save_of_step = h->d_save_of_step;
        a.du0 = ddu0; a.dp_members = ddp; a.partials = h->d_partials; a.dp = ddp; a.ticket = h->d_ticket;
        a.N = c.N; a.Npad = h->Npad; a.S = h->S; a.tb = h->tb; a.trace = h->d_trace;
        for (int j = 0; j < 4; j++) { a.cost_a[j] = h->cost_av[j]; a.cost_b[j] = h->cost_bv[j]; a.cont_a[j] = h->cont_av[j]; a.cont_b[j] = h->cont_bv[j]; }
        a.flags = ((c.flags & B200ADJ_FLAG_NO_START) ? 1u : 0u) | ((c.flags & B200ADJ_FLAG_NO_CHECKPOINTING) ? 2u : 0u) |
                  ((c.flags & B200ADJ_FLAG_CKPT_EVERY_STEP) ? 4u : 0u) | (h->cont_on ? 8u : 0u);
        switch (c.rhs_family) {
        case B200ADJ_FAM_LV: rc = launch_rev<LotkaVolterra>(h, a); break;
        case B200ADJ_FAM_LORENZ: rc = launch_rev<Lorenz>(h, a); break;
        case B200ADJ_FAM_ROBERTSON: rc = launch_rev<Robertson>(h, a); break;
        default: { const FamilyVTable* vt = family_lookup(c.rhs_family); rc = (vt && vt->rev) ? vt->rev(h, a) : B200ADJ_ERR_UNSUPPORTED; }
        }
    } else {
        SdeRevArgs a;
        a.ckpt = h->d_ckpt; a.p = h->cur_p; a.dLdu = dL; a.save_of_step = h->d_save_of_step;
        a.du0 = ddu0; a.dp_members = ddp; a.partials = h->d_partials; a.dp = ddp; a.ticket = h->d_ticket;
        a.N = c.N; a.S = h->S; a.h = c.dt;
        for (int j = 0; j < 4; j++) { a.cost_a[j] = h->cost_av[j]; a.cost_b[j] = h->cost_bv[j]; }
        a.flags = ((c.flags & B200ADJ_FLAG_NO_START) ? 1u : 0u) | ((c.flags & B200ADJ_FLAG_NO_CHECKPOINTING) ? 2u : 0u) | ((c.flags & B200ADJ_FLAG_CKPT_EVERY_STEP) ? 4u : 0u);
        a.seed = c.seed; a.traj_offset = c.traj_offset;
        a.noise = h->noise_valid ? h->d_noise : nullptr;
        rc = sde_reverse_dispatch(h, a);
    }
    if (rc) { h->err = "reverse dispatch failed (sensealg/family not built)"; return rc; }
    CUDA_TRY(h, cudaGetLastError());
    // parameter part of the cost family (dgdp_discrete at every applied jump, dgdp_continuous over the horizon): independent of
    // the state, so it joins dp after the reverse kernels (ReverseLossCallback src/adjoint_common.jl:771-783, accumulate_cost!
    // src/derivative_wrappers.jl:1411-1442, QuadratureAdjoint src/quadrature_adjoint.jl:547-553, 601-605)
    if (h->has_dgdp || (h->has_cdgdp && h->cont_on)) {
        DgdpArgs g;
        memset(&g, 0, sizeof(g));
        int njump = c.K;
        if ((c.flags & B200ADJ_FLAG_NO_START) && c.sensealg != B200ADJ_SA_BACKSOLVE && c.K > 0 && h->saveat[0] == c.t0) njump--;
        for (int q = 0; q < 8; q++) {
            g.c[q] = (h->has_dgdp ? njump * h->dgdp_c[q] : 0.0) + ((h->has_cdgdp && h->cont_on) ? (c.t1 - c.t0) * h->cdgdp_c[q] : 0.0);
            g.e[q] = (h->has_dgdp ? njump * h->dgdp_e[q] : 0.0) + ((h->has_cdgdp && h->cont_on) ? (c.t1 - c.t0) * h->cdgdp_e[q] : 0.0);
        }
        g.p = h->cur_p; g.dp = ddp; g.N = c.N; g.P = c.P; g.shared_p = c.shared_p; g.f32 = c.dtype != B200ADJ_F64;
        const int64_t work = c.shared_p ? 1 : c.N;
        dgdp_add_kernel<<<(unsigned)((work + 127) / 128), 128, 0, h->stream>>>(g);
        h->launches++;
        CUDA_TRY(h, cudaGetLastError());
    }
    // multi-GPU: the ONE collective of the path -- dG/dp summed over the ranks (shared parameters only; SURVEY.md 8e)
    if (c.shared_p && h->nranks > 1 && !fused_allreduce) { rc = comm_allreduce(h, ddp, (size_t)c.P); if (rc) return rc; }
    if (!c.buffers_on_device) {
        CUDA_TRY(h, cudaMemcpyAsync(du0, h->s_du0, c.d * N * e, cudaMemcpyDeviceToHost, h->stream));
        CUDA_TRY(h, cudaMemcpyAsync(dp, h->s_dp, pn * e, cudaMemcpyDeviceToHost, h->stream));
        CUDA_TRY(h, cudaStreamSynchronize(h->stream));
    }
    return B200ADJ_OK;
}

int32_t b200adj_get_noise(void* handle, void* dW_out) {
    if (!handle || !dW_out) return B200ADJ_ERR_INVALID;
    Handle* h = (Handle*)handle;
    const b200adj_cfg& c = h->cfg;
    if (!is_sde(c) || !h->have_forward) { h->err = "no SDE forward pass to report"; return B200ADJ_ERR_STATE; }
    CUDA_TRY(h, cudaSetDevice(c.device));
    const size_t bytes = (size_t)h->S * c.m * (size_t)c.N * esz(c);
    if (!h->noise_valid) {
        // regenerate from the Philox counter into the handle's buffer
        SdeNoiseArgs a; a.out = h->d_noise; a.N = c.N; a.S = h->S; a.h = c.dt; a.seed = c.seed; a.traj_offset = c.traj_offset; a.m = c.m;
        const int64_t total = (int64_t)h->S * c.N;
        sde_noise_launch(h, a, total);
        CUDA_TRY(h, cudaGetLastError());
    }
    CUDA_TRY(h, cudaMemcpyAsync(dW_out, h->d_noise, bytes, c.buffers_on_device ? cudaMemcpyDeviceToDevice : cudaMemcpyDeviceToHost, h->stream));
    CUDA_TRY(h, cudaStreamSynchronize(h->stream));
    return B200ADJ_OK;
}

int32_t b200adj_get_block_trace(void* handle, uint64_t* out, int32_t* nblocks) {
    if (!handle || !nblocks) return B200ADJ_ERR_INVALID;
    Handle* h = (Handle*)handle;
    *nblocks = h->grid;
    if (!out) return B200ADJ_OK;
    if (!h->d_trace) { h->err = "handle was not created with B200ADJ_FLAG_TRACE"; return B200ADJ_ERR_STATE; }
    CUDA_TRY(h, cudaSetDevice(h->cfg.device));
    CUDA_TRY(h, cudaStreamSynchronize(h->stream));
    CUDA_TRY(h, cudaMemcpy(out, h->d_trace, (size_t)h->grid * 3 * sizeof(unsigned long long), cudaMemcpyDeviceToHost));
    return B200ADJ_OK;
}

int32_t b200adj_destroy(void* handle) {
    if (!handle) return B200ADJ_ERR_INVALID;
    Handle* h = (Handle*)handle;
    cudaSetDevice(h->cfg.device);
    cudaStreamSynchronize(h->stream);
    comm_release(h);
    free_all(h);
    delete h;
    return B200ADJ_OK;
}

}  // extern "C"
