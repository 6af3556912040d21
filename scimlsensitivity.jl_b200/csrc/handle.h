// handle.h -- the state behind one b200adj handle and the kernel-dispatch entry points shared by the translation
// units of libb200adj.so.  api.cu owns the C ABI (include/b200adj.h); every disp_*.cu instantiates the kernels of one
// stepper (x one RHS family) so the library builds in parallel.
#pragma once
#include <cuda_runtime.h>
#include <math.h>
#include <stdint.h>
#include <stdio.h>
#include <string.h>
#include <stdlib.h>

#include <string>
#include <type_traits>
#include <unordered_map>
#include <vector>

#include "../../include/b200adj.h"
#include "ode_tsit5.cuh"
#include "sde_em.cuh"
#include "ros23.cuh"
#include "mlp.cuh"
#include "tsit5_quad.cuh"
#include "mlp_tc.cuh"
#include "mlp_tc_wide.cuh"
#include "tsit5_adaptive.cuh"

namespace b200adj {

// Which kernel framework serves a handle; decided once by b200adj_create.
enum class Path {
    FIXED,      // fixed-step Tsit5 on the dt grid (ode_tsit5.cuh, tsit5_quad.cuh; F64, and F32 for LV / Lorenz)
    T5A,        // per-member dense Tsit5 (tsit5_adaptive.cuh): adaptive, or fixed step with off-grid save times
    ROS,        // Rosenbrock23 (ros23.cuh)
    SDE,        // Euler-Maruyama / Euler-Heun (sde_em.cuh)
    MLP         // neural ODE family (mlp.cuh; BF16_F32ACC: mlp_tc.cuh, mlp_tc_wide.cuh)
};

struct Handle {
    b200adj_cfg cfg;
    Path path = Path::FIXED;
    std::vector<double> saveat;
    std::vector<int32_t> save_of_step;
    int S = 0;
    int64_t Npad = 0;
    int block = 64, grid = 0, nsm = 132;
    int ckpt_every = 1;               // fixed-step Tsit5: forward states kept every C steps, segments re-solved in the reverse pass
    cudaStream_t stream = nullptr, own_stream = nullptr;
    // device memory owned by the handle
    double* d_ckpt = nullptr;         // [S/C+1][d][Npad]
    double* d_noise = nullptr;        // [S][m][N] (SDE, stored-noise mode)
    double* d_partials = nullptr;     // [grid][P]
    double* d_adj_dense = nullptr;    // QuadratureAdjoint, fixed-step Tsit5: [S][8][d][Npad]
    unsigned long long* d_trace = nullptr;   // [grid][3] block trace (B200ADJ_FLAG_TRACE)
    unsigned int* d_ticket = nullptr;
    int32_t* d_save_of_step = nullptr;
    int maxs = 0;                     // T5A / ROS: per-member step capacity of the dense forward / reverse solutions (T5A with
                                      // B200ADJ_FLAG_CHECKPOINT_SAVES: of ONE save interval)
    // T5A, B200ADJ_FLAG_CHECKPOINT_SAVES: the checkpoint of every save interval, [N][ck_nseg][2 d + 4] (tsit5_adaptive.cuh,
    // t5a_ckpt); the intervals are bounded by t0, the save times inside (t0, t1) -- saveat[ck_k0 ..] -- and t1
    double* d_ck = nullptr; int ck_nseg = 0, ck_k0 = 0;
    double adj_abstol = 0, adj_reltol = 0;   // <= 0: use the forward tolerances
    // named cost family, per component (b200adj_set_cost_family; the scalar entry points broadcast):
    //   discrete (COST_AFFINE)  dgdu = cost_av .* u + cost_bv,  dgdp = dgdp_c .* p + dgdp_e   at every save time
    //   continuous              dgdu = cont_av .* u + cont_bv,  dgdp = cdgdp_c .* p + cdgdp_e
    bool cont_on = false;
    double cost_av[4] = {0, 0, 0, 0}, cost_bv[4] = {0, 0, 0, 0}, cont_av[4] = {0, 0, 0, 0}, cont_bv[4] = {0, 0, 0, 0};
    bool has_dgdp = false, has_cdgdp = false;
    double dgdp_c[8] = {0}, dgdp_e[8] = {0}, cdgdp_c[8] = {0}, cdgdp_e[8] = {0};
    float* d_kst = nullptr;           // tensor-core MLP path: the forward stages of every step ([S][7][2][N] floats)
    double *r_ft = nullptr, *r_fu = nullptr, *r_fk = nullptr, *d_saveat = nullptr;
    // QuadratureAdjoint on T5A / ROS (allocated at the first Quadrature reverse pass): member-major reverse dense solution +
    // member-major copy of the forward one (quadgk.cuh)
    double *r_rrec = nullptr, *r_rend = nullptr, *r_ftT = nullptr, *r_frecT = nullptr;
    int32_t *r_fn = nullptr, *r_rn = nullptr;
    // quadgk scratch of the QuadratureAdjoint kernels, sized per RESIDENT warp of the persistent grid qgrid (quadgk.cuh)
    double *r_qseg = nullptr, *r_qkey = nullptr; int maxseg = 0; int qgrid = 0; size_t qpartials_blocks = 0;
    // forward save table (the primal output of b200adj_forward) kept apart from the reverse pass' jump times
    int fwd_K = 0; std::vector<double> fwd_saveat; std::vector<int32_t> fwd_save_of_step; int32_t* d_fwd_save_of_step = nullptr; double* d_fwd_saveat = nullptr;
    // staging (buffers_on_device == 0)
    double *s_u0 = nullptr, *s_p = nullptr, *s_saved = nullptr, *s_dLdu = nullptr, *s_du0 = nullptr, *s_dp = nullptr, *s_dW = nullptr;
    int32_t* s_status = nullptr;
    int32_t* r_status = nullptr;      // T5A: per-member status of the last forward pass, whether or not the caller asked for it (the reverse pass reads it)
    const double* cur_p = nullptr;    // device pointer to p valid between forward and reverse
    int32_t* d_ev_ac = nullptr; int32_t* d_ev_ak = nullptr; double* d_ev_af = nullptr;      // b200adj_set_event_param_shift
    int32_t* d_event_of_step = nullptr;     // fixed-step Tsit5: event index at grid point n, or -1
    int nev = 0; double *d_ev_t = nullptr, *d_ev_s = nullptr, *d_ev_c = nullptr, *d_ev_ps = nullptr, *d_ev_pc = nullptr;      // preset-time events
    // state-dependent event (b200adj_set_continuous_callback): per-member event lists cc_t[cc_maxev][N], cc_n[N] and the
    // event words cc_ev[cc_maxev][N] of the events found
    bool cc_on = false; int cc_idx = 0, cc_dir = 0, cc_pcomp = -1, cc_pparam = 0, cc_maxev = 0;
    double cc_level = 0, cc_psign = 1, cc_scale[4] = {1, 1, 1, 1}, cc_shift[4] = {0, 0, 0, 0};
    int cc_lparam = -1, cc_acomp = -1, cc_aparam = 0, cc_qcomp = -1; double cc_lcoef = 0, cc_acoef = 0, cc_qcoef = 1;      // b200adj_set_continuous_callback_params
    double* d_cc_t = nullptr; int32_t* d_cc_n = nullptr; int32_t* d_cc_ev = nullptr;
    // the callback's family mode (b200adj_set_family_events): fe_nc > 0 conditions of the family and their directions
    int fe_nc = 0; int32_t fe_dir[8] = {0};
    int rev_block = 0; const void* rev_block_kernel = nullptr;      // adaptive Tsit5 reverse kernel: block size chosen per instantiation (disp_t5a.inc)
    bool have_forward = false;
    bool noise_valid = false;
    int64_t launches = 0;
    Tsit5Tables tb;
    // multi-GPU (comm.cu): one NCCL communicator per handle, dp all-reduced on the handle's stream
    void* nccl_comm = nullptr; int nranks = 1, rank = 0;
    // fused all-reduce over peer memory (ode_tsit5.cuh::reduce_dp): this handle's mailbox, the peers' mailboxes mapped here
    P2PComm p2p = {};                 // p2p.nranks > 1 once the mailboxes are exchanged
    void* p2p_mailbox = nullptr;      // owned
    void* p2p_ipc_open[P2P_MAXRANKS] = {nullptr};   // cudaIpcOpenMemHandle mappings to close
    unsigned long long p2p_epoch = 0;
    std::string err;
    // the device memory the handle owns (b200adj_device_bytes): every allocation goes through dev_malloc / dev_free
    int64_t dev_bytes = 0;
    std::unordered_map<const void*, size_t> dev_sizes;
};

template <class T> cudaError_t dev_malloc(Handle* h, T** p, size_t bytes) {
    const cudaError_t e = cudaMalloc((void**)p, bytes);
    if (e == cudaSuccess) { h->dev_sizes[*p] = bytes; h->dev_bytes += (int64_t)bytes; }
    return e;
}
template <class T> void dev_free(Handle* h, T*& p) {
    if (!p) return;
    const auto it = h->dev_sizes.find(p);
    if (it != h->dev_sizes.end()) { h->dev_bytes -= (int64_t)it->second; h->dev_sizes.erase(it); }
    cudaFree((void*)p);
    p = nullptr;
}

#define CUDA_TRY(h, expr)                                                                      \
    do {                                                                                       \
        cudaError_t _e = (expr);                                                               \
        if (_e != cudaSuccess) {                                                               \
            (h)->err = std::string(#expr) + ": " + cudaGetErrorString(_e);                     \
            return B200ADJ_ERR_CUDA;                                                           \
        }                                                                                      \
    } while (0)

// ---- kernel dispatch (disp_*): a runtime choice becomes a std::integral_constant passed to the generic lambda f, whose
// body names the kernel instantiation with X.value ----
template <class F> int with_flag(bool b, F&& f) { return b ? f(std::true_type{}) : f(std::false_type{}); }
template <class F> int with_cost(const Handle* h, F&& f) {
    if (h->cfg.cost_kind == B200ADJ_COST_EXPLICIT) return f(std::integral_constant<int, COST_EXPLICIT>{});
    return f(std::integral_constant<int, COST_AFFINE>{});
}
template <class F> int with_sensealg(int32_t sensealg, F&& f) {
    switch (sensealg) {
    case B200ADJ_SA_INTERPOLATING: return f(std::integral_constant<int, SA_INTERP>{});
    case B200ADJ_SA_GAUSS: return f(std::integral_constant<int, SA_GAUSS>{});
    case B200ADJ_SA_BACKSOLVE: return f(std::integral_constant<int, SA_BACKSOLVE>{});
    case B200ADJ_SA_GAUSSKRONROD: return f(std::integral_constant<int, SA_GK>{});
    case B200ADJ_SA_QUADRATURE: return f(std::integral_constant<int, SA_QUAD>{});
    default: return B200ADJ_ERR_UNSUPPORTED;
    }
}
// One launch on the handle's stream.  Static shared memory rides on top of the dynamic `smem`, so the kernel opts in to
// more dynamic shared memory well below the 48 KB default limit.
template <class... P, class... A>
int launch_kernel(Handle* h, void (*kernel)(P...), dim3 grid, dim3 block, size_t smem, const A&... args) {
    if (smem > 30 * 1024 && cudaFuncSetAttribute(kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem) != cudaSuccess) return B200ADJ_ERR_CUDA;
    kernel<<<grid, block, smem, h->stream>>>(args...);
    h->launches++;
    return 0;
}

inline bool is_sde(const b200adj_cfg& c) { return c.stepper == B200ADJ_ST_EM || c.stepper == B200ADJ_ST_EULER_HEUN; }
inline bool is_adaptive(const Handle* h) { return h->path == Path::T5A || h->path == Path::ROS; }
// T5A run with a constant step and no error control (fixed-step Tsit5 with off-grid save times)
inline bool is_fixed_dt(const Handle* h) { return h->path == Path::T5A && h->cfg.stepper == B200ADJ_ST_TSIT5_FIXED; }
inline bool is_mlp_tc(const Handle* h) { return h->path == Path::MLP && h->cfg.dtype == B200ADJ_BF16_F32ACC; }
// the kernels' `flags` word (KF_* bits, ode_tsit5.cuh)
inline uint32_t kernel_flags(const Handle* h) {
    const uint32_t f = h->cfg.flags;
    return ((f & B200ADJ_FLAG_NO_START) ? KF_NO_START : 0u) | ((f & B200ADJ_FLAG_NO_CHECKPOINTING) ? KF_NO_CHECKPOINTING : 0u) |
           ((f & B200ADJ_FLAG_CKPT_EVERY_STEP) ? KF_CKPT_EVERY_STEP : 0u) | (h->cont_on ? KF_CONT_COST : 0u) |
           (is_fixed_dt(h) ? KF_FIXED_DT : 0u);
}
inline size_t esz(const b200adj_cfg& c) { return c.dtype == B200ADJ_F64 ? sizeof(double) : sizeof(float); }   // BF16_F32ACC: fp32 buffers at the ABI

void tsit5_weights(double th, double* w, double (*Rout)[4] = nullptr);
void build_tsit5_tables(double h, Tsit5Tables* t);
void build_c4_du_weights(double h, double* w);     // OdeRevArgsT::hC4u
void hermite_thetas(double* th);                   // the 7 theta of Tsit5Tables::hHm and OdeRevArgsT::hHf
void build_hermite_folded(double h, double (*hf)[4]);   // OdeRevArgsT::hHf
// OdeRevArgsT<float>::hC4u and hHf: the fp64 weights, each rounded once to float
inline void build_hermite_weights_f32(double h, float* c4u, float (*hf)[4]) {
    double w[7], f[7][4];
    build_c4_du_weights(h, w);
    build_hermite_folded(h, f);
    for (int j = 0; j < 7; j++) c4u[j] = (float)w[j];
    for (int r = 0; r < 7; r++) for (int j = 0; j < 4; j++) hf[r][j] = (float)f[r][j];
}
template <class T, class S> inline void cast_tables(const S& src, T* dst) {
    for (int i = 0; i < 7; i++) for (int j = 0; j < 6; j++) dst->hA[i][j] = (float)src.hA[i][j];
    for (int i = 0; i < 4; i++) for (int j = 0; j < 7; j++) dst->hBst[i][j] = (float)src.hBst[i][j];
    for (int i = 0; i < 3; i++) for (int j = 0; j < 7; j++) dst->hBq[i][j] = (float)src.hBq[i][j];
    for (int i = 0; i < 3; i++) dst->hGW[i] = (float)src.hGW[i];
    for (int i = 0; i < 7; i++) for (int j = 0; j < 4; j++) dst->hHm[i][j] = (float)src.hHm[i][j];
    for (int j = 0; j < 7; j++) dst->hR4[j] = (float)src.hR4[j];
}


// ---- family registry (SURVEY.md 8f rank 4; the seam user-supplied ODEFunction(f; vjp, vjp_p, jac, paramjac) occupies in the
// reference, src/derivative_wrappers.jl:284-359, test/Core3/user_vjp.jl:14-38).  A family PLUG-IN is a shared library built from
// a user header that defines one struct with the shape of families.cuh (D, P, f, vjp_u, vjp_p [, jac, djac, dvjp_p]), or for a
// diagonal-noise SDE one `template <bool ITO> struct` with the shape of SdeLotkaVolterra (D, P, M = D, f, g and their VJPs),
// or for a general-noise SDE one plain struct (D, P, M, f and its VJPs, and the contractions g_apply / gvjp_u_apply /
// gvjp_p_apply of its D x M diffusion with the increments; sde_em.cuh);
// the plug-in instantiates the same kernel templates for it and exports this table of launchers (family_plugin.inc).
// b200adj_register_family(path) loads it and hands out a family id >= B200ADJ_FAM_USER_BASE.  The built-in families fill
// the same table (api.cu, builtin_families), so every family dispatches through one lookup (the MLP family's row has no
// launchers: Path::MLP has its own, mlp_*_dispatch). ----
struct FamilyVTable {
    uint32_t abi;                 // B200ADJ_PLUGIN_ABI of the headers the plug-in was built from
    int32_t d, P;
    const char* name;
    int (*fwd)(Handle*, const OdeFwdArgs&);          // fixed-step Tsit5
    int (*rev)(Handle*, const OdeRevArgs&);
    int (*t5a_fwd)(Handle*, const T5aArgs&);         // adaptive Tsit5 / dense fixed-step framework
    int (*t5a_rev)(Handle*, const T5aArgs&);
    int (*ros_fwd)(Handle*, const RosArgs&);         // Rosenbrock23 (null when the family has no jac / djac / dvjp_p)
    int (*ros_rev)(Handle*, const RosArgs&);
    int (*fwd_f32)(Handle*, const OdeFwdArgsT<float>&);     // fixed-step Tsit5 in F32 (built-in LV / Lorenz; null elsewhere)
    int (*rev_f32)(Handle*, const OdeRevArgsT<float>&);
    int32_t nc;                   // conditions of the family's own state-dependent event (B200ADJ_FAMILY_HAS_EVENTS); 0: none
    int32_t m;                    // Wiener processes of an SDE family (diagonal noise: m = d); 0: an ODE family
    int32_t noise;                // B200ADJ_NOISE_*: NONE for an ODE family, DIAGONAL or GENERAL for an SDE family
    int (*sde_fwd)(Handle*, const SdeFwdArgs&);      // EM / EulerHeun (SDE families only; null for an ODE family)
    int (*sde_rev)(Handle*, const SdeRevArgs&);
};
constexpr uint32_t B200ADJ_PLUGIN_ABI = 0x00030000u ^ (uint32_t)sizeof(Handle) ^ ((uint32_t)sizeof(OdeRevArgs) << 8) ^
                                        ((uint32_t)sizeof(T5aArgs) << 16) ^ ((uint32_t)sizeof(FamilyVTable) << 24) ^
                                        ((uint32_t)sizeof(SdeFwdArgs) << 4) ^ ((uint32_t)sizeof(SdeRevArgs) << 12);
constexpr int B200ADJ_FAM_USER_BASE_ID = 100;
// api.cu: the families, built-in (id < B200ADJ_FAM_USER_BASE_ID) and registered plug-ins; null for an unknown id
const FamilyVTable* family_lookup(int id);

// ---- dispatch entry points, one explicit instantiation per family in disp_*.cu ----
template <class Fam> int launch_fwd(Handle* h, const OdeFwdArgs& a);
template <class Fam> int launch_rev(Handle* h, const OdeRevArgs& a);
template <class Fam> int launch_fwd_f32(Handle* h, const OdeFwdArgsT<float>& a);
template <class Fam> int launch_rev_f32(Handle* h, const OdeRevArgsT<float>& a);
template <class Fam> int launch_t5a_fwd(Handle* h, const T5aArgs& a);
template <class Fam> int launch_t5a_rev(Handle* h, const T5aArgs& a);
template <class Fam> int launch_ros_fwd(Handle* h, const RosArgs& a);
template <class Fam> int launch_ros_rev(Handle* h, const RosArgs& a);
template <template <bool> class Fam> int launch_sde_fwd(Handle* h, const SdeFwdArgs& a);     // disp_sde.inc
template <template <bool> class Fam> int launch_sde_rev(Handle* h, const SdeRevArgs& a);
int sde_noise_launch(Handle* h, const SdeNoiseArgs& a, int64_t total);
int mlp_forward_dispatch(Handle* h, const void* u0, const void* p, void* saved, int32_t* status);
int mlp_reverse_dispatch(Handle* h, const void* dLdu, void* du0, void* dp);
int comm_allreduce(Handle* h, void* buf, size_t count);     // comm.cu: in-place sum over ranks on h->stream (no-op without a communicator)
void comm_release(Handle* h);
bool comm_fused_ready(const Handle* h);    // the peer mailboxes of the fused all-reduce are mapped

// persistent grid of the quadrature kernels and the dynamic shared memory (block maxima of the key array) per block
inline int quad_grid(int64_t N, int nsm) { const int64_t g = (N + QUAD_WARPS - 1) / QUAD_WARPS, cap = (int64_t)nsm * QUAD_BLOCKS_PER_SM; return (int)(g < cap ? g : cap); }
// blocks actually launched: what is resident at once (a static member -> warp assignment must not queue a second, partial wave)
template <class K> inline int quad_launch_grid(const Handle* h, K kernel, size_t smem) {
    int nb = 0;
    if (smem > 32 * 1024) cudaFuncSetAttribute(kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem);   // static smem rides on top
    if (cudaOccupancyMaxActiveBlocksPerMultiprocessor(&nb, kernel, QUAD_WARPS * 32, smem) != cudaSuccess || nb < 1) nb = 1;
    const int cap = nb * h->nsm;
    return h->qgrid < cap ? h->qgrid : cap;
}
int ensure_quad_buffers(Handle* h);      // api.cu: lazily allocates QuadratureAdjoint's dense solutions and the quadgk scratch
inline size_t quad_smem(int maxseg) { return (size_t)QUAD_WARPS * (QUAD_SKEYS + quad_l1_blocks(maxseg)) * sizeof(double); }
inline size_t quad_seg_doubles(int P, int maxseg, int qgrid) { return (size_t)qgrid * QUAD_WARPS * maxseg * (size_t)(((P + 4 + 3) / 4) * 4); }
// QuadratureAdjoint on every stepper: its buffers, then `rev` (the stepper's SA_QUAD reverse pass, which stores the dense
// reverse solution; on Rosenbrock23 also the member-major copy of the forward one), then the quadrature kernel kernel(SP)
// over the persistent grid with the arguments args(), taken once the buffers exist
template <class Rev, class Kernel, class Args>
int quadrature_adjoint(Handle* h, Rev&& rev, Kernel&& kernel, Args&& args) {
    if (int rc = ensure_quad_buffers(h)) return rc;
    if (int rc = rev()) return rc;
    if ((size_t)h->qgrid > h->qpartials_blocks) return B200ADJ_ERR_INVALID;
    const auto a = args();
    const size_t smem = quad_smem(h->maxseg);
    return with_flag(h->cfg.shared_p, [&](auto SP) {
        const auto k = kernel(SP);
        k<<<quad_launch_grid(h, k, smem), QUAD_WARPS * 32, smem, h->stream>>>(a);
        h->launches++;
        return 0;
    });
}

}  // namespace b200adj
