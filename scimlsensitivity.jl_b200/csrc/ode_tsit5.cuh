// ode_tsit5.cuh -- fixed-step Tsit5 ensemble kernels: forward solve with per-step checkpoints and the fused
// reverse (adjoint) pass.  One ensemble member per thread, SoA [step][dim][member] so every global access is a
// fully coalesced 8 B x 32 lanes = 256 B row; the whole time loop runs inside the kernel so lambda, the dG/dp
// accumulators and the FSAL stages never leave registers (SURVEY.md 7.2 item 1: a per-step launch would be
// launch-latency bound at N = 65536).  The body of one loop iteration is exactly "one fused reverse time step":
//   checkpoint load -> forward-stage recompute (dense output data) -> interpolate y at the 6 adjoint stage times
//   -> batched RHS + VJPs -> Tsit5 stage update -> 3-pt Gauss dG/dp accumulate -> jump at save times.
//
// Reference functions replaced (per stage, per member):
//   sense functors   src/interpolating_adjoint.jl:150-174, src/gauss_adjoint.jl:118-128, src/backsolve_adjoint.jl:32-61
//   split_states     sol(y,t,continuity=:right)  src/interpolating_adjoint.jl:190-205, src/gauss_adjoint.jl:158-166
//   vecjacobian!     src/derivative_wrappers.jl:256-267         vec_pjac!  src/gauss_adjoint.jl:629-743
//   GaussIntegrand   src/gauss_adjoint.jl:745-759 (+ upstream IntegratingSumCallback, 3-pt Gauss-Legendre per step)
//   ReverseLossCallback  src/adjoint_common.jl:754-821 (lambda += dgdu at t_k, FSAL k1 recomputed)
//   backsolve_checkpoint_callbacks  src/backsolve_adjoint.jl:523-546
// and the upstream Tsit5 perform_step! / dense interpolant (SURVEY.md App. B).
//
// Arithmetic notes.  (1) The step size is folded into the tableau on the host (hA = h*A, hBst = h*b(theta_s),
// hBq = h*b(theta_q)) and the tables travel as kernel PARAMETERS, i.e. they sit in the constant bank and feed DFMA
// directly as c[][] operands: one FMA per tableau entry, no register cost, no __constant__ symbol shared between
// handles.  (2) The adjoint derivative is carried with the opposite sign, ka' = +J'lam, so that the reverse step
// lam + (-h) * sum a_sj (-J'lam_j) becomes lam + sum hA_sj ka'_j with the SAME table as the forward stages.
#pragma once
#include <cuda_runtime.h>
#include <stdint.h>
#include "families.cuh"
#include "quadgk.cuh"

namespace b200adj {

// R = real type of the solve: double (all paths) or float (the fp32 throughput variant of the fixed-step ODE path)
template <class R> struct Tsit5TablesT {
    R hA[7][6];    // h * A[s][j] (row 6 = h * b)
    R hBst[4][7];  // h * b_j(theta) at theta = 1 - c_s for adjoint stages s = 1..4 (0-based)
    R hBq[3][7];   // h * b_j(theta) at theta = (1 -/+ sqrt(.6))/2, 1/2  (3-pt Gauss-Legendre nodes)
    R hGW[3];      // (h/2) * Gauss-Legendre weights 5/9, 8/9, 5/9
    // Hermite form of the forward dense output: per point {H01, h*H10, h*H11, theta^2 (1-theta)^2} at the 4 adjoint stage
    // times (rows 0..3, theta of hBst) and at the y-side Gauss nodes (rows 4..6: row 4 + g has the theta of hBq[2 - g]), and
    // hR4 = h * (theta^4 coefficient of b_j).  The reverse kernel reads the same points with c4's elimination folded in
    // (OdeRevArgsT::hHf)
    R hHm[7][4];
    R hR4[7];
};
using Tsit5Tables = Tsit5TablesT<double>;

// mailboxes of the fused cross-GPU all-reduce of dG/dp (see reduce_dp below)
constexpr int P2P_PMAX = 8, P2P_MAXRANKS = 8;
struct P2PComm {
    double* slots[P2P_MAXRANKS];              // slots[r]: mailbox of rank r as seen from this device
    unsigned long long* flags[P2P_MAXRANKS];  // flags[r]: epoch counters of rank r's mailbox
    int32_t nranks, rank;                     // nranks <= 1: not used
    unsigned long long epoch;                 // this gradient's epoch (1, 2, ...: every rank launches the same sequence)
};

enum { SA_INTERP = 0, SA_GAUSS = 1, SA_QUAD = 2, SA_BACKSOLVE = 3, SA_GK = 4 };
enum { COST_EXPLICIT = 0, COST_AFFINE = 1 };

template <class R> struct OdeFwdArgsT {
    const R* u0;        // [D][N]
    const R* p;         // [P] or [P][N]
    R* ckpt;            // [S+1][D][N]
    R* saved;           // [K][D][N] or null
    const int32_t* save_of_step;  // [S+1]: save index k at grid point n, or -1
    int32_t* status;         // [N] or null
    int64_t N;
    int64_t Npad;            // checkpoint row pitch: N rounded up to the block size (every block owns full 16B-aligned rows)
    int32_t S;
    int32_t ckpt_every;      // C: row m of ckpt holds u_{mC} (m < ceil(S/C)), row ceil(S/C) holds u_S; C = 1: every step
    // preset-time events on the dt grid (EV kernels): event_of_step[n] = e when the affect u <- ev_s[e] .* u + ev_c[e]
    // (and p <- ev_ps[e] .* p + ev_pc[e]) fires at t_n, else -1
    const int32_t* event_of_step; const double* ev_s; const double* ev_c; const double* ev_ps; const double* ev_pc; int32_t nev;
    Tsit5TablesT<R> tb;
};
using OdeFwdArgs = OdeFwdArgsT<double>;

// bits of the kernels' `flags` word (OdeRevArgsT, T5aArgs, RosArgs, SdeRevArgs, MlpArgs); handle.h::kernel_flags builds it
constexpr uint32_t KF_NO_START = 1u;            // no loss jump at t0 (B200ADJ_FLAG_NO_START)
constexpr uint32_t KF_NO_CHECKPOINTING = 2u;    // BacksolveAdjoint(checkpointing = false)
constexpr uint32_t KF_CKPT_EVERY_STEP = 4u;     // Backsolve: checkpoints at every step instead of the save times
constexpr uint32_t KF_CONT_COST = 8u;           // continuous cost: dlam -= dgdu_continuous(y)
constexpr uint32_t KF_FIXED_DT = 16u;           // T5A kernels: constant step dt0, no error control

template <class R> struct OdeRevArgsT {
    const R* ckpt;      // [S+1][D][N]
    const R* p;         // [P] or [P][N]
    const R* dLdu;      // [K][D][N] (COST_EXPLICIT)
    const int32_t* save_of_step;
    R* du0;             // [D][N]
    R* dp_members;      // [P][N] when !shared_p
    double* partials;        // [gridDim][P] block partial sums (shared_p)
    R* dp;              // [P] final (shared_p)
    unsigned int* ticket;    // last-block-done counter
    int64_t N;
    int64_t Npad;            // checkpoint row pitch
    int32_t S;
    int32_t slots;           // member slots per block (= checkpoint tile width); blockDim.x > slots => the top warp row rotates
    int32_t ckpt_every;      // C > 1 (SEG kernels): forward states kept every C steps, each segment re-solved into shared memory
    R cost_a[4], cost_b[4];   // COST_AFFINE, per component: dgdu_discrete = cost_a .* u(t_k) + cost_b
    R cont_a[4], cont_b[4];   // continuous cost g = sum_j cont_a_j/2 u_j^2 + cont_b_j u_j:  dlam -= dgdu_continuous(y)  (KF_CONT_COST)
    uint32_t flags;          // KF_* bits
    R* adj_dense;       // SA_QUAD: [S][8][D][Npad] = (lambda at the start of reverse step n, ka'[0..6]) per step
    unsigned long long* trace;   // optional [gridDim][3] = (smid, globaltimer at block start, at block end) or null
    const int32_t* event_of_step; const double* ev_s; const double* ev_c; const double* ev_ps; const double* ev_pc; int32_t nev;   // EV kernels
    R Rpoly[7][4];               // SA_GK: dense-output polynomials b_j(theta) = sum_m Rpoly[j][m] theta^(m+1)
    R hstep;                     // SA_GK: the step size
    R hC4u[7];                   // c4 weights of k1..k5, of du (slot 5, in place of k6) and of k7 (tsit5_hermite_c4_du reads 1..4)
    R hHf[7][4];                 // tsit5_dense_hermite: hHm's points with the c4 elimination folded in (build_hermite_folded)
    P2PComm p2p;                 // fused cross-GPU all-reduce of dp (nranks <= 1: off)
    Tsit5TablesT<R> tb;
};
using OdeRevArgs = OdeRevArgsT<double>;

template <int D, class R> __device__ __forceinline__ void load_state(const R* base, int64_t N, int64_t i, R* u) {
#pragma unroll
    for (int j = 0; j < D; j++) u[j] = __ldg(base + (int64_t)j * N + i);
}
template <int D, class R> __device__ __forceinline__ void store_state(R* base, int64_t N, int64_t i, const R* u) {
#pragma unroll
    for (int j = 0; j < D; j++) base[(int64_t)j * N + i] = u[j];
}

// ---- TMA (bulk async copy) + mbarrier primitives: HBM -> shared memory staging of the forward checkpoints ----
// SASS: UBLKCP.S.G (cp.async.bulk) / SYNCS.ARRIVE.TRANS64 (expect_tx) / SYNCS.PHASECHK (try_wait).
__device__ __forceinline__ uint32_t smem_u32(const void* p) { return (uint32_t)__cvta_generic_to_shared(p); }
__device__ __forceinline__ void mbar_init(uint64_t* bar, uint32_t count) {
    asm volatile("mbarrier.init.shared::cta.b64 [%0], %1;" ::"r"(smem_u32(bar)), "r"(count) : "memory");
}
__device__ __forceinline__ void mbar_fence_init() { asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory"); }
__device__ __forceinline__ void mbar_expect_tx(uint64_t* bar, uint32_t bytes) {
    asm volatile("mbarrier.arrive.expect_tx.shared::cta.b64 _, [%0], %1;" ::"r"(smem_u32(bar)), "r"(bytes) : "memory");
}
__device__ __forceinline__ void tma_load_1d(void* dst_smem, const void* src_gmem, uint32_t bytes, uint64_t* bar) {
    asm volatile("cp.async.bulk.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1], %2, [%3];"
                 ::"r"(smem_u32(dst_smem)), "l"(src_gmem), "r"(bytes), "r"(smem_u32(bar)) : "memory");
}
__device__ __forceinline__ void mbar_wait(uint64_t* bar, uint32_t parity) {
    asm volatile(
        "{\n"
        ".reg .pred p;\n"
        "LAB_WAIT%=:\n"
        "mbarrier.try_wait.parity.shared::cta.b64 p, [%0], %1;\n"
        "@p bra LAB_DONE%=;\n"
        "bra LAB_WAIT%=;\n"
        "LAB_DONE%=:\n"
        "}\n" ::"r"(smem_u32(bar)), "r"(parity) : "memory");
}

// stage value  u + sum_{j<S_} hA[S_][j] k_j
template <int D, int S_, class R> __device__ __forceinline__ void tsit5_stage(const Tsit5TablesT<R>& tb, const R* u, const R (*k)[D], R* out) {
#pragma unroll
    for (int i = 0; i < D; i++) {
        R acc = u[i];
#pragma unroll
        for (int j = 0; j < S_; j++) acc = fma(tb.hA[S_][j], k[j][i], acc);
        out[i] = acc;
    }
}
// dense output  u + sum_j w[j] k_j   (w already scaled by h)
template <int D, class R> __device__ __forceinline__ void tsit5_dense(const R* u, const R (*k)[D], const R* w, R* out) {
#pragma unroll
    for (int i = 0; i < D; i++) {
        R acc = u[i];
#pragma unroll
        for (int j = 0; j < 7; j++) acc = fma(w[j], k[j][i], acc);
        out[i] = acc;
    }
}
// The same dense output in Hermite form.  The Tsit5 interpolant is a C1 Hermite quartic: b_j(1) = b_j (row 6 of hA / h),
// b_j'(0) = delta_j1, b_j'(1) = delta_j7, so with du = u_{n+1} - u_n, k1, k7 = f(u_{n+1}) and c4 = sum_j hR4[j] k_j
//   y(theta) = u_n + H01 du + h H10 k1 + h H11 k7 + theta^2 (1-theta)^2 c4
// (H01 = 3t^2 - 2t^3, H10 = t - 2t^2 + t^3, H11 = t^3 - t^2).  u_{n+1} and k7 must be the end point of the SAME step as k1..k6.
// k6 need not be formed: u_{n+1} = u_n + sum_{j<6} hA[6][j] k_j (b7 = 0), so k6 = (du - sum_{j<5} hA[6][j] k_j) / hA[6][5]
// and c4 = sum_{j<5} w_j k_j + w_5 du + hR4[6] k7 with w_j = hR4[j] - hR4[5] b_j / b6 and w_5 = R4[5] / b6 (build_c4_du_weights).
// The w_0 k1, w_5 du and w_6 k7 terms then fold into the point weights (build_hermite_folded, a row of OdeRevArgsT::hHf):
//   y(theta) = u_n + (H01 + G w_5) du + (h H10 + G w_0) k1 + (h H11 + G w_6) k7 + G c4'',   c4'' = sum_{j=1..4} w_j k_j
// with G = theta^2 (1-theta)^2 <= 1/16: 3 D ops for c4'' (tsit5_hermite_c4_du) and 4 D FMAs per point (tsit5_dense_hermite),
// against 7 D per point for tsit5_dense.  A reverse step that has u_{n+1} from the forward pass then rebuilds stages 2..5
// only.  du carries the rounding of the forward step's sum (about one ulp of u), which |H01 + G w_5| <= 1 + 15/16 passes
// on to y.  The identity is one of the tableau alone, so it holds for the adjoint step's own dense output as well (u_n ->
// lambda at the step's start, du -> the step's increment, k -> its stages ka').
template <int D, class R>
__device__ __forceinline__ void tsit5_hermite_c4_du(const R* w, const R (*k)[D], R* c4) {
#pragma unroll
    for (int i = 0; i < D; i++) {
        R acc = w[1] * k[1][i];
#pragma unroll
        for (int j = 2; j < 5; j++) acc = fma(w[j], k[j][i], acc);
        c4[i] = acc;
    }
}
template <int D, class R>
__device__ __forceinline__ void tsit5_dense_hermite(const R* u, const R* du, const R* k1, const R* k7, const R* c4, const R* w, R* out) {
#pragma unroll
    for (int i = 0; i < D; i++) out[i] = fma(w[3], c4[i], fma(w[2], k7[i], fma(w[1], k1[i], fma(w[0], du[i], u[i]))));
}

// producer/consumer named barriers (ids 1..15; id 0 is __syncthreads)
__device__ __forceinline__ void named_bar_sync(int id, int nthreads) { asm volatile("bar.sync %0, %1;" ::"r"(id), "r"(nthreads) : "memory"); }
__device__ __forceinline__ void named_bar_arrive(int id, int nthreads) { asm volatile("bar.arrive %0, %1;" ::"r"(id), "r"(nthreads) : "memory"); }

// ------------------------------------------------------------------------------------------------------------
// Forward ensemble solve, fixed-step Tsit5, writes every step's state (the dense solution is NOT stored: the
// reverse pass recomputes the 6 stages from u_n, 24 B/step instead of 192 B/step of HBM traffic).
// ------------------------------------------------------------------------------------------------------------
// parameters in force after the first `upto` events (p0 = the caller's parameters of this member)
template <int P, class R>
__device__ __forceinline__ void fixed_event_params(const double* ev_ps, const double* ev_pc, int upto, const R* p0, R* p) {
#pragma unroll
    for (int q = 0; q < P; q++) p[q] = p0[q];
    if (!ev_ps) return;
    for (int e = 0; e < upto; e++) {
#pragma unroll
        for (int q = 0; q < P; q++) p[q] = (R)ev_ps[e * P + q] * p[q] + (R)ev_pc[e * P + q];
    }
}

template <class Fam, bool SHARED_P, class R = double, bool EV = false>
__global__ void __launch_bounds__(512) tsit5_forward_kernel(const __grid_constant__ OdeFwdArgsT<R> a) {
    constexpr int D = Fam::D, P = Fam::P;
    const int64_t gi = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
    const bool active = gi < a.N;
    const int64_t i = active ? gi : a.N - 1;
    R p[P];
#pragma unroll
    for (int q = 0; q < P; q++) p[q] = SHARED_P ? __ldg(a.p + q) : __ldg(a.p + (int64_t)q * a.N + i);
    R u[D], k[7][D], tmp[D];
    load_state<D>(a.u0, a.N, i, u);
    const int64_t stride = (int64_t)D * a.N, cstride = (int64_t)D * a.Npad;
    const int CK = a.ckpt_every > 1 ? a.ckpt_every : 1;
    // checkpoints: padded pitch, threads past N shadow member N-1 and fill the pad columns (keeps TMA rows whole)
    store_state<D>(a.ckpt, a.Npad, gi, u);
    if (active && a.saved) { int ks = a.save_of_step[0]; if (ks >= 0) store_state<D>(a.saved + (int64_t)ks * stride, a.N, i, u); }
    Fam::f(u, p, k[0]);
    // (travelling warp groups as in the reverse kernel were tried here: the extra control flow of the free-running loop
    // costs more than the rotation gains, so the forward kernel launches `slots` threads)
    for (int n = 0; n < a.S; n++) {
        tsit5_stage<D, 1>(a.tb, u, k, tmp); Fam::f(tmp, p, k[1]);
        tsit5_stage<D, 2>(a.tb, u, k, tmp); Fam::f(tmp, p, k[2]);
        tsit5_stage<D, 3>(a.tb, u, k, tmp); Fam::f(tmp, p, k[3]);
        tsit5_stage<D, 4>(a.tb, u, k, tmp); Fam::f(tmp, p, k[4]);
        tsit5_stage<D, 5>(a.tb, u, k, tmp); Fam::f(tmp, p, k[5]);
        tsit5_stage<D, 6>(a.tb, u, k, tmp);
#pragma unroll
        for (int j = 0; j < D; j++) u[j] = tmp[j];
        if (EV) {
            // preset-time event at t_{n+1}: u <- s .* u + c, p <- ps .* p + pc (PresetTimeCallback, save_positions = (false,
            // false)); the checkpoint and a coinciding save point record the POST-event state, FSAL is recomputed from it
            const int e = a.event_of_step[n + 1];
            if (e >= 0 && n + 1 < a.S) {
#pragma unroll
                for (int j = 0; j < D; j++) u[j] = (R)a.ev_s[e * D + j] * u[j] + (R)a.ev_c[e * D + j];
                if (a.ev_ps) {
#pragma unroll
                    for (int q = 0; q < P; q++) p[q] = (R)a.ev_ps[e * P + q] * p[q] + (R)a.ev_pc[e * P + q];
                }
            }
        }
        Fam::f(u, p, k[0]);                      // FSAL: k7 of this step = k1 of the next
        // checkpoints: every step, or every C-th step plus the final state (CheckpointSolution grid of the reference,
        // src/interpolating_adjoint.jl:54-112: the reverse pass re-solves each segment from its left checkpoint)
        if (CK == 1) store_state<D>(a.ckpt + (int64_t)(n + 1) * cstride, a.Npad, gi, u);
        else if ((n + 1) % CK == 0) store_state<D>(a.ckpt + (int64_t)((n + 1) / CK) * cstride, a.Npad, gi, u);
        else if (n + 1 == a.S) store_state<D>(a.ckpt + (int64_t)((a.S + CK - 1) / CK) * cstride, a.Npad, gi, u);
        if (active && a.saved) { int ks = a.save_of_step[n + 1]; if (ks >= 0) store_state<D>(a.saved + (int64_t)ks * stride, a.N, i, u); }
    }
    if (active && a.status) {
        bool ok = true;
#pragma unroll
        for (int j = 0; j < D; j++) ok = ok && isfinite(u[j]);
        a.status[i] = ok ? 0 : 1;
    }
}

// ---- fused all-reduce of dG/dp over the GPUs of one box (SURVEY.md 8e: "fuse the last reverse-step block reduction with the
// allreduce") ----  Every rank owns a MAILBOX in its HBM: slots[2 parities][nranks][P2P_PMAX] doubles + flags[nranks] epoch
// counters, mapped into every peer (CUDA IPC / peer access over NVLink; comm.cu).  The last block of the reverse kernel
// writes its dG/dp into slot [rank] of EVERY mailbox (peer stores), publishes the epoch in every mailbox' flags[rank]
// (st.release.sys), waits until its own mailbox shows the epoch from all ranks (ld.acquire.sys) and sums the slots in rank
// order -- the same bits on every rank, no collective kernel, no extra launch.
__device__ __forceinline__ void st_release_sys(unsigned long long* p, unsigned long long v) { asm volatile("st.release.sys.global.u64 [%0], %1;" ::"l"(p), "l"(v) : "memory"); }
__device__ __forceinline__ unsigned long long ld_acquire_sys(const unsigned long long* p) { unsigned long long v; asm volatile("ld.acquire.sys.global.u64 %0, [%1];" : "=l"(v) : "l"(p) : "memory"); return v; }
__device__ __forceinline__ double ld_relaxed_sys_f64(const double* p) { double v; asm volatile("ld.relaxed.sys.global.f64 %0, [%1];" : "=d"(v) : "l"(p) : "memory"); return v; }

// deterministic block reduction of P per-thread values -> partials[block][P]; the last block to finish sums the
// partials in index order (fixed order => bitwise reproducible for a given grid), no floating-point atomics.
// pc (optional): the fused cross-GPU all-reduce above.
template <int P, class RO>
__device__ __forceinline__ void reduce_dp(const double* acc, double* partials, RO* dp, unsigned int* ticket, const P2PComm* pc = nullptr) {
    __shared__ double s_red[16 * P];               // up to 512 threads per block
    const int nwarps = (int)(blockDim.x >> 5);
    __shared__ bool s_last;
    const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
#pragma unroll
    for (int q = 0; q < P; q++) {
        double v = acc[q];
#pragma unroll
        for (int off = 16; off > 0; off >>= 1) v += __shfl_xor_sync(0xffffffffu, v, off);
        if (lane == 0) s_red[warp * P + q] = v;
    }
    __syncthreads();
    if (threadIdx.x < P) {
        double v = 0.0;
        for (int w = 0; w < nwarps; w++) v += s_red[w * P + threadIdx.x];
        partials[(int64_t)blockIdx.x * P + threadIdx.x] = v;
    }
    __threadfence();
    __syncthreads();
    if (threadIdx.x == 0) {
        unsigned int t = atomicAdd(ticket, 1u);
        s_last = (t == gridDim.x - 1);
    }
    __syncthreads();
    if (s_last) {
        __threadfence();
        // P x gridDim sums; each warp-lane strides over blocks in a fixed pattern, then a fixed shuffle tree
        for (int q = warp; q < P; q += nwarps) {
            double v = 0.0;
            for (unsigned int b = lane; b < gridDim.x; b += 32) v += __ldcg(partials + (int64_t)b * P + q);
#pragma unroll
            for (int off = 16; off > 0; off >>= 1) v += __shfl_xor_sync(0xffffffffu, v, off);
            if (lane == 0) {
                if (pc && pc->nranks > 1) {
                    const int par = (int)(pc->epoch & 1ull);
                    for (int r = 0; r < pc->nranks; r++) pc->slots[r][(size_t)(par * pc->nranks + pc->rank) * P2P_PMAX + q] = v;     // peer stores
                } else dp[q] = (RO)v;
            }
        }
        if (pc && pc->nranks > 1) {
            __syncthreads();                      // every slot of this rank is on its way
            if (threadIdx.x == 0) {
                __threadfence_system();
                for (int r = 0; r < pc->nranks; r++) st_release_sys(pc->flags[r] + pc->rank, pc->epoch);
                bool ok = true;
                const long long t0 = clock64();
                for (int r = 0; r < pc->nranks; r++)
                    while (ld_acquire_sys(pc->flags[pc->rank] + r) < pc->epoch) {
                        if (clock64() - t0 > 8000000000LL) { ok = false; break; }      // ~4 s: a peer that never launched -- fail loudly
                    }
                s_last = ok;                      // reuse: false => poison the result
            }
            __syncthreads();
            if (threadIdx.x < P) {
                const int par = (int)(pc->epoch & 1ull);
                double tot = 0.0;
                for (int r = 0; r < pc->nranks; r++) tot += ld_relaxed_sys_f64(pc->slots[pc->rank] + (size_t)(par * pc->nranks + r) * P2P_PMAX + threadIdx.x);
                dp[threadIdx.x] = s_last ? (RO)tot : (RO)__longlong_as_double(0x7ff8000000000000LL);
            }
        }
        if (threadIdx.x == 0) *ticket = 0;   // re-arm for the next launch
    }
}

// dG/dp write-out of a reverse kernel: a shared p sums acc over the grid (reduce_dp; an inactive thread adds zeros, and every
// thread of the block must arrive), a per-member p stores member i's row.
template <int P, bool SHARED_P>
__device__ __forceinline__ void store_dp(double* acc, bool active, int64_t i, int64_t N, double* dp_members, double* partials, double* dp,
                                         unsigned int* ticket) {
    if (SHARED_P) {
        if (!active) {
#pragma unroll
            for (int q = 0; q < P; q++) acc[q] = 0.0;
        }
        reduce_dp<P>(acc, partials, dp, ticket);
    } else if (active) {
#pragma unroll
        for (int q = 0; q < P; q++) dp_members[(int64_t)q * N + i] = acc[q];
    }
}

// Body of the three QuadratureAdjoint kernels (tsit5_quad.cuh, tsit5_adaptive.cuh, ros23.cuh), which differ only in `make(i)`,
// member i's integrand context: quad_member_loop over the members, per-member dp stored as each member finishes, a shared p
// summed over the grid (lane 0 of each warp carries its members' sum).  Here rather than next to quad_member_loop because
// quadgk.cuh comes before reduce_dp.
template <int P, bool SHARED_P, class Args, class MAKE>
__device__ __forceinline__ void quad_kernel_body(const Args& a, const MAKE& make) {
    extern __shared__ double s_quad_l1[];
    const int lane = threadIdx.x & 31;
    double acc[P];
#pragma unroll
    for (int q = 0; q < P; q++) acc[q] = 0.0;
    auto sink = [&](int64_t i, const double* res) {
        if (SHARED_P) {
#pragma unroll
            for (int q = 0; q < P; q++) acc[q] += res[q];
        } else if (lane == 0) {
#pragma unroll
            for (int q = 0; q < P; q++) a.dp_members[(int64_t)q * a.N + i] = res[q];
        }
    };
    quad_member_loop<P>(a.N, a.K, a.saveat, a.t0, a.t1, a.quad_abstol, a.quad_reltol, a.qseg, a.qkey, a.maxseg, s_quad_l1, make, sink);
    if (SHARED_P) store_dp<P, true>(acc, lane == 0, 0, a.N, a.dp_members, a.partials, a.dp, a.ticket);
}

// accumulate_cost! (src/derivative_wrappers.jl:1411-1442): with ka' = -dlam/dt the continuous cost adds +dgdu_continuous(y)
template <int D, bool CONT, class Args, class R>
__device__ __forceinline__ void add_continuous(const Args& a, const R* y, R* ka) {
    if (CONT) {
#pragma unroll
        for (int j = 0; j < D; j++) ka[j] += fma(a.cont_a[j], y[j], a.cont_b[j]);
    }
}

template <int D, int COST, class Args, class R>
__device__ __forceinline__ void add_cotangent(const Args& a, int ks, int64_t stride, int64_t N, int64_t i, const R* y, R* lam) {
    if (COST == COST_EXPLICIT) {
#pragma unroll
        for (int j = 0; j < D; j++) lam[j] += __ldg(a.dLdu + (int64_t)ks * stride + (int64_t)j * N + i);
    } else {
#pragma unroll
        for (int j = 0; j < D; j++) lam[j] += fma(a.cost_a[j], y[j], a.cost_b[j]);
    }
}

// ------------------------------------------------------------------------------------------------------------
// Fused reverse pass.  SA in {SA_INTERP, SA_GAUSS, SA_BACKSOLVE}.
// Register cap: 65536 members / 132 SMs (H100 SXM) = 497 threads per SM must be resident at once, otherwise a second,
// nearly empty wave doubles the kernel time (every thread runs the full time loop): 512 threads/SM => <= 128 registers.
// ------------------------------------------------------------------------------------------------------------
#ifndef B200_REV_MAXREG
#define B200_REV_MAXREG 128
#endif
#ifndef REV_CH_DEF
#define REV_CH_DEF 4
#endif
constexpr int REV_CH = REV_CH_DEF, REV_NST = 2;     // TMA pipeline: steps per stage (= block barrier period), stages in flight
static_assert(REV_CH_DEF <= 4, "hand-over barrier ids are keyed by step & 3: the block barrier period must not exceed 4 steps");
template <int D, class R = double> constexpr size_t rev_smem_bytes(int block) { return (size_t)REV_NST * REV_CH * D * block * sizeof(R); }
// SEG kernels (interval checkpointing): one re-solved segment of C states per member slot instead of the TMA stages
template <int D, class R = double> constexpr size_t rev_seg_smem_bytes(int block, int C) { return (size_t)C * D * block * sizeof(R); }
template <class Fam, int SA, bool SHARED_P, int COST, bool CONT, class R = double, bool SEG = false, bool EV = false>
__global__ void __maxnreg__(B200_REV_MAXREG) tsit5_reverse_kernel(const __grid_constant__ OdeRevArgsT<R> a) {
    constexpr int D = Fam::D, P = Fam::P;
    // BLOCK = member slots of this block.  When the slot count is not a multiple of 4 warps the SM's four sub-partitions
    // (one fp64 pipe each; warp w lives on sub-partition w % 4) would carry unequal warp counts for the whole solve:
    // 448 slots = 4,4,3,3 warps, and the kernel runs at the pace of the 4-warp sub-partitions.  The host then launches whole warp rows
    // (blockDim.x = 128 * ceil(BLOCK / 128)) and the rw = (BLOCK / 32) % 4 warp groups of the top row travel round the
    // four sub-partitions, one hop per time step: group q4+e is advanced through step c by warp q4 + ((e + c) & 3), which
    // takes the group's live state from its predecessor through shared memory (producer/consumer named barriers) and
    // hands it on after the step.  Every sub-partition then carries q4/4 + rw/4 warps of work on average.
    const int BLOCK = a.slots;
    const bool rot = (int)blockDim.x > BLOCK;
    const int wid = (int)(threadIdx.x >> 5), q4 = (BLOCK >> 7) << 2, rw = (BLOCK >> 5) & 3;
    const bool top = rot && wid >= q4;
    auto group_of = [&](int c) -> int {           // member group this warp advances through step counter c (-1: resting)
        if (!top) return wid;
        const int e = ((wid - q4) - c) & 3;
        return e < rw ? q4 + e : -1;
    };
    int grp = group_of(0);
    // global member index of this thread's current slot (the group changes per step for the travelling warps)
    auto member_gi = [&]() -> int64_t { return (int64_t)blockIdx.x * BLOCK + grp * 32 + (int)(threadIdx.x & 31); };
    auto member_i = [&]() -> int64_t { const int64_t g = member_gi(); return (grp >= 0 && g < a.N) ? g : a.N - 1; };
    int64_t gi = member_gi();
    bool active = grp >= 0 && gi < a.N;
    int64_t i = active ? gi : a.N - 1;
    const int64_t N = a.N, stride = (int64_t)D * N, Npad = a.Npad, cstride = (int64_t)D * Npad;
    const Tsit5TablesT<R>& tb = a.tb;
    if (a.trace && threadIdx.x == 0) {
        unsigned int smid; unsigned long long t;
        asm volatile("mov.u32 %0, %%smid;" : "=r"(smid));
        asm volatile("mov.u64 %0, %%globaltimer;" : "=l"(t));
        a.trace[blockIdx.x * 3 + 0] = smid; a.trace[blockIdx.x * 3 + 1] = t;
    }
    R p[P];
#pragma unroll
    for (int q = 0; q < P; q++) p[q] = SHARED_P ? __ldg(a.p + q) : __ldg(a.p + (int64_t)q * N + i);

    if (EV && a.ev_ps) {               // the reverse solve starts on the last segment: parameters after all events
        R p0[P];
#pragma unroll
        for (int q = 0; q < P; q++) p0[q] = p[q];
        fixed_event_params<P>(a.ev_ps, a.ev_pc, a.nev, p0, p);
    }
    // reverse affect of a preset-time event at t_n (after the checkpoint reset and the loss jump of the same time):
    // lam(tau-) = s .* lam(tau+), dG/dp scaled by ps, parameters of the segment below re-derived from the caller's p
    auto reverse_affect = [&](int e, R* lam_, R* mu_, int64_t mi) {
#pragma unroll
        for (int j = 0; j < D; j++) lam_[j] *= (R)a.ev_s[e * D + j];
        if (a.ev_ps) {
#pragma unroll
            for (int q = 0; q < P; q++) mu_[q] *= (R)a.ev_ps[e * P + q];
            R p0[P];
#pragma unroll
            for (int q = 0; q < P; q++) p0[q] = SHARED_P ? __ldg(a.p + q) : __ldg(a.p + (int64_t)q * N + mi);
            fixed_event_params<P>(a.ev_ps, a.ev_pc, e, p0, p);
        }
    };
    R lam[D], mu[P];                 // mu: dG/dp accumulator (Gauss quadrature sum, or the augmented state)
#pragma unroll
    for (int j = 0; j < D; j++) lam[j] = 0.0;
#pragma unroll
    for (int q = 0; q < P; q++) mu[q] = 0.0;

    if (SA == SA_BACKSOLVE) {
        // z = [lam; mu; y]; dy/dt = f(y) integrated backwards (src/backsolve_adjoint.jl:32-61).
        // ky' = -f(y), kl' = +J'lam so that both use the +h tables.
        R y[D];
        load_state<D>(a.ckpt + (int64_t)a.S * cstride, Npad, gi, y);
        { int ks = a.save_of_step[a.S]; if (ks >= 0) add_cotangent<D, COST>(a, ks, stride, N, i, y, lam); }
        R ky[7][D], kl[7][D], ys[D], ls[D], dg[P];
        const bool ckpt_on = !(a.flags & KF_NO_CHECKPOINTING), every = (a.flags & KF_CKPT_EVERY_STEP);
        bool fsal = false;
        for (int n = a.S - 1; n >= 0; n--) {
            if (!fsal) {
                Fam::f(y, p, ky[0]);
#pragma unroll
                for (int j = 0; j < D; j++) ky[0][j] = -ky[0][j];
                Fam::vjp_u(y, p, lam, kl[0]);
                add_continuous<D, CONT>(a, y, kl[0]);
            }
            Fam::vjp_p(y, p, lam, dg);                 // mu' = -F'lam, reverse step: mu += h * sum b_j F'(y_j) lam_j
#pragma unroll
            for (int q = 0; q < P; q++) mu[q] = fma(tb.hA[6][0], dg[q], mu[q]);
#define B200_BS_STAGE(S_)                                                                 \
            tsit5_stage<D, S_>(tb, y, ky, ys); tsit5_stage<D, S_>(tb, lam, kl, ls);       \
            Fam::f(ys, p, ky[S_]);                                                        \
            _Pragma("unroll") for (int j = 0; j < D; j++) ky[S_][j] = -ky[S_][j];         \
            Fam::vjp_u(ys, p, ls, kl[S_]); add_continuous<D, CONT>(a, ys, kl[S_]);              \
            if (S_ < 6) { Fam::vjp_p(ys, p, ls, dg);                                      \
                _Pragma("unroll") for (int q = 0; q < P; q++) mu[q] = fma(tb.hA[6][S_ < 6 ? S_ : 0], dg[q], mu[q]); }
            B200_BS_STAGE(1) B200_BS_STAGE(2) B200_BS_STAGE(3) B200_BS_STAGE(4) B200_BS_STAGE(5) B200_BS_STAGE(6)
#undef B200_BS_STAGE
            // after stage 6: ys, ls hold the new state (c7 = 1, row 6 = b), ky[6], kl[6] are the FSAL derivatives
#pragma unroll
            for (int j = 0; j < D; j++) { y[j] = ys[j]; lam[j] = ls[j]; ky[0][j] = ky[6][j]; kl[0][j] = kl[6][j]; }
            fsal = true;
            // callbacks at t_n: checkpoint reset first, then the loss jump (CallbackSet order, backsolve_adjoint.jl:545);
            // no_start never skips the jump for Backsolve (src/adjoint_common.jl:761)
            const int ks = a.save_of_step[n];
            if (ckpt_on && (every || ks >= 0)) { load_state<D>(a.ckpt + (int64_t)n * cstride, Npad, gi, y); fsal = false; }
            if (ks >= 0) { add_cotangent<D, COST>(a, ks, stride, N, i, y, lam); fsal = false; }
            if (EV) {
                const int e = a.event_of_step[n];
                if (e >= 0 && n > 0) {
                    reverse_affect(e, lam, mu, i);
                    // y(tau-): the forward step below the event, re-solved from its checkpoint with the pre-event parameters
                    // (the reference keeps it as `uleft` of the tracked affect)
                    R ub[D], kk[7][D], tt_[D];
                    load_state<D>(a.ckpt + (int64_t)(n - 1) * cstride, Npad, gi, ub);
                    Fam::f(ub, p, kk[0]);
                    tsit5_stage<D, 1>(tb, ub, kk, tt_); Fam::f(tt_, p, kk[1]);
                    tsit5_stage<D, 2>(tb, ub, kk, tt_); Fam::f(tt_, p, kk[2]);
                    tsit5_stage<D, 3>(tb, ub, kk, tt_); Fam::f(tt_, p, kk[3]);
                    tsit5_stage<D, 4>(tb, ub, kk, tt_); Fam::f(tt_, p, kk[4]);
                    tsit5_stage<D, 5>(tb, ub, kk, tt_); Fam::f(tt_, p, kk[5]);
                    tsit5_stage<D, 6>(tb, ub, kk, y);
                    fsal = false;
                }
            }
        }
    } else {
        R kf[7][D];                       // forward stages of the current step; kf[6] = f(u_{n+1}) carried over
        R ka[7][D];                       // adjoint stages (+J'lam); ka[0] carried over (FSAL) unless a jump hit
        R ulo[D], uhi[D];                 // u_n, u_{n+1} (the end point of the Hermite dense output)
        // Forward checkpoints are staged HBM -> shared memory by TMA bulk copies, CH steps per stage, NST stages in
        // flight, completion tracked by one mbarrier per stage.  A register prefetch does not survive the register
        // cap (ptxas sinks the LDG next to its use and every step then eats a full DRAM latency -- 32% of all
        // warp-stall samples in the first ncu profile); the async copy cannot be sunk and costs no registers.
        // The block-wide barrier that recycles a stage every CH steps also keeps all warps of the SM in lockstep: the
        // warp arbiter favours high warp ids, and free-running warps drift apart by >2x over the 1000 steps (block
        // trace: 0.94 .. 2.2 ms for identical work) so the stragglers finish latency-bound; per-warp pipelines with
        // a coarse barrier measured slower as well (2.12-2.21 ms vs 1.98 ms) -- lockstep warps share the I-cache.
        constexpr int CH = REV_CH, NST = REV_NST;
        extern __shared__ __align__(128) unsigned char s_ck_raw[];
        R* const s_ck = reinterpret_cast<R*>(s_ck_raw);      // [NST][CH][D][BLOCK]
        __shared__ __align__(8) uint64_t s_bar[NST];
        const uint32_t row_bytes = (uint32_t)(BLOCK * sizeof(R));      // BLOCK % 32 == 0 => a multiple of 16 B in both precisions
        const int NC = (a.S + CH - 1) / CH;    // chunk k holds steps n = S-1-(k*CH+j), j = 0..CH-1
        const R* ck_col = a.ckpt + (int64_t)blockIdx.x * BLOCK;
        auto issue_chunk = [&](int k) {
            const int st = k % NST;
            const int cnt = min(CH, a.S - k * CH);
            mbar_expect_tx(&s_bar[st], (uint32_t)(cnt * D) * row_bytes);
            for (int j = 0; j < cnt; j++) {
                const int nn = a.S - 1 - (k * CH + j);
#pragma unroll
                for (int dd = 0; dd < D; dd++)
                    tma_load_1d(&s_ck[(size_t)((st * CH + j) * D + dd) * BLOCK], ck_col + ((int64_t)nn * D + dd) * Npad, row_bytes, &s_bar[st]);
            }
        };
        if (!SEG) {
            if (threadIdx.x == 0) {
                for (int st = 0; st < NST; st++) mbar_init(&s_bar[st], 1);
                mbar_fence_init();
            }
            __syncthreads();
            if (threadIdx.x == 0) for (int k = 0; k < NST && k < NC; k++) issue_chunk(k);
        }
        // SEG (checkpoint_every = C > 1; CheckpointSolution machinery of src/interpolating_adjoint.jl:54-112, 206-278 and
        // src/gauss_adjoint.jl:57-95, 167-212): only u_{mC} is in HBM.  When the reverse solve enters segment m (its first step
        // is n = min((m+1)C, S) - 1) the member's forward solve is repeated from u_{mC} and the C states land in this slot's
        // own shared-memory column; the steps of the segment then read them back exactly as the TMA path reads its tile.
        const int CK = SEG ? a.ckpt_every : 1;
        const int MROW = SEG ? (a.S + CK - 1) / CK : a.S;          // checkpoint row holding u_S

        constexpr int NV = 4 * D + P;          // rotating state: lam, mu, ka[0], kf[6], uhi
        __shared__ R s_mig[3 * NV * 32];
        __shared__ R s_migp[SHARED_P ? 1 : 3 * P * 32];          // per-member parameters of the travelling groups
        if (!SHARED_P && top && grp >= 0) {
#pragma unroll
            for (int q = 0; q < P; q++) s_migp[((grp - q4) * P + q) * 32 + (threadIdx.x & 31)] = p[q];
        }
        load_state<D>(a.ckpt + (int64_t)MROW * cstride, Npad, grp >= 0 ? gi : 0, uhi);
        {
            // jump at t = T (PresetTimeCallback fires at initialisation when T is a save time)
            int ks = a.save_of_step[a.S];
            if (ks >= 0) add_cotangent<D, COST>(a, ks, stride, N, i, uhi, lam);
            Fam::f(uhi, p, kf[6]);
            Fam::vjp_u(uhi, p, lam, ka[0]);    // y(T) = u_S
            add_continuous<D, CONT>(a, uhi, ka[0]);
        }
        bool need_left = false;
        for (int n = a.S - 1; n >= 0; n--) {
            const int c = a.S - 1 - n, k = c / CH, jj = c % CH, st = k % NST;
            if (top) {
                const int lane = (int)(threadIdx.x & 31);
                grp = group_of(c);
                if (c > 0 && grp >= 0) {       // take the group over from the warp that advanced it through step c-1
                    // barrier id keyed by (group, step & 3): resting warps run ahead of the group by up to one barrier
                    // window (CH = 4 steps), so consecutive hand-overs of one group must not share an id
                    named_bar_sync(1 + (grp - q4) * 4 + (c & 3), 64);
                    const R* m = s_mig + (size_t)(grp - q4) * NV * 32 + lane;
#pragma unroll
                    for (int j = 0; j < D; j++) { lam[j] = m[j * 32]; ka[0][j] = m[(D + j) * 32]; kf[6][j] = m[(2 * D + j) * 32]; uhi[j] = m[(3 * D + j) * 32]; }
#pragma unroll
                    for (int q = 0; q < P; q++) mu[q] = m[(4 * D + q) * 32];
                    if (!SHARED_P) {
#pragma unroll
                        for (int q = 0; q < P; q++) p[q] = s_migp[((grp - q4) * P + q) * 32 + lane];
                    }
                }
            }
            if (!SEG) {
                if (jj == 0) mbar_wait(&s_bar[st], (uint32_t)((k / NST) & 1));
                if (grp >= 0) {
#pragma unroll
                    for (int dd = 0; dd < D; dd++) ulo[dd] = s_ck[(size_t)((st * CH + jj) * D + dd) * BLOCK + grp * 32 + (threadIdx.x & 31)];
                }
                if (jj == CH - 1 || n == 0) {
                    __syncthreads();               // every thread has read this stage: hand it back to the TMA producer
                    if (threadIdx.x == 0 && k + NST < NC) issue_chunk(k + NST);
                }
            } else {
                const int m = n / CK, js = n - m * CK;
                const int slot = grp * 32 + (int)(threadIdx.x & 31);
                if (grp >= 0 && (n == a.S - 1 || js == CK - 1)) {
                    // entering segment m: forward re-solve u_{mC} -> u_{mC + cnt - 1} into this slot's column
                    const int cnt = min(CK, a.S - m * CK);
                    R us[D], ts[D];
                    load_state<D>(a.ckpt + (int64_t)m * cstride, Npad, member_gi(), us);
#pragma unroll
                    for (int dd = 0; dd < D; dd++) s_ck[(size_t)dd * BLOCK + slot] = us[dd];
                    Fam::f(us, p, kf[0]);
                    for (int q = 1; q < cnt; q++) {
                        tsit5_stage<D, 1>(tb, us, kf, ts); Fam::f(ts, p, kf[1]);
                        tsit5_stage<D, 2>(tb, us, kf, ts); Fam::f(ts, p, kf[2]);
                        tsit5_stage<D, 3>(tb, us, kf, ts); Fam::f(ts, p, kf[3]);
                        tsit5_stage<D, 4>(tb, us, kf, ts); Fam::f(ts, p, kf[4]);
                        tsit5_stage<D, 5>(tb, us, kf, ts); Fam::f(ts, p, kf[5]);
                        tsit5_stage<D, 6>(tb, us, kf, ts);
#pragma unroll
                        for (int dd = 0; dd < D; dd++) { us[dd] = ts[dd]; s_ck[(size_t)(q * D + dd) * BLOCK + slot] = ts[dd]; }
                        Fam::f(us, p, kf[0]);
                    }
                }
                if (grp >= 0) {
#pragma unroll
                    for (int dd = 0; dd < D; dd++) ulo[dd] = s_ck[(size_t)(js * D + dd) * BLOCK + slot];
                }
                if (jj == CH - 1 || n == 0) __syncthreads();       // lockstep only (see above)
            }
            if (grp < 0) continue;             // resting warp of the rotating row: barriers only

            // ---- forward stage recompute on [t_n, t_{n+1}]: the dense-output data of this step ----
            // k6 only where something needs more than the Hermite data: GaussKronrod's general-theta dense output and the
            // event kernels' left limit (stage 6 re-derived); the Hermite points take du in its place (tsit5_hermite_c4_du)
            constexpr bool K6 = SA == SA_GK;
            R tmp[D];
            Fam::f(ulo, p, kf[0]);
            tsit5_stage<D, 1>(tb, ulo, kf, tmp); Fam::f(tmp, p, kf[1]);
            tsit5_stage<D, 2>(tb, ulo, kf, tmp); Fam::f(tmp, p, kf[2]);
            tsit5_stage<D, 3>(tb, ulo, kf, tmp); Fam::f(tmp, p, kf[3]);
            tsit5_stage<D, 4>(tb, ulo, kf, tmp); Fam::f(tmp, p, kf[4]);
            if (K6 || (EV && need_left)) { tsit5_stage<D, 5>(tb, ulo, kf, tmp); Fam::f(tmp, p, kf[5]); }

            if (EV && need_left) {
                // the step above ended with an event at t_{n+1}: the first adjoint stage sees the LEFT limit there -- the end
                // state of this forward step (pre-event), its k7 = f(u-) and the adjoint derivative at (u-, lam-)
                tsit5_stage<D, 6>(tb, ulo, kf, uhi);
                Fam::f(uhi, p, kf[6]);
                Fam::vjp_u(uhi, p, lam, ka[0]);
                add_continuous<D, CONT>(a, uhi, ka[0]);
                need_left = false;
            }
            // Hermite data of the forward dense output: uhi / kf[6] are this step's end point (the checkpoint u_{n+1} and its
            // FSAL derivative, or the re-derived left limit at an event, so du is this step's own increment); kf[1..5] are
            // dead from here on (except for GK)
            R du[D], c4[D];
#pragma unroll
            for (int j = 0; j < D; j++) du[j] = uhi[j] - ulo[j];
            tsit5_hermite_c4_du<D>(a.hC4u, kf, c4);
#ifdef REV_MIDSYNC
            __syncthreads();
#endif
            // ---- adjoint Tsit5 step t_{n+1} -> t_n; stage s evaluated at y(t_{n+1} - c_s h) ----
            R ls[D], y[D], dg[P];
            if (SA == SA_INTERP) {
                // mu' = -F'lam integrated with the same tableau: mu += h * sum_j b_j F'(y_j) lam_j ; stage 1 at y = u_{n+1}
                Fam::vjp_p(uhi, p, lam, dg);
#pragma unroll
                for (int q = 0; q < P; q++) mu[q] = fma(tb.hA[6][0], dg[q], mu[q]);
            }
#define B200_ADJ_STAGE(S_, YEXPR)                                                          \
            tsit5_stage<D, S_>(tb, lam, ka, ls);                                           \
            YEXPR;                                                                         \
            Fam::vjp_u(y, p, ls, ka[S_]); add_continuous<D, CONT>(a, y, ka[S_]);                 \
            if (SA == SA_INTERP && S_ < 6) { Fam::vjp_p(y, p, ls, dg);                     \
                _Pragma("unroll") for (int q = 0; q < P; q++) mu[q] = fma(tb.hA[6][S_ < 6 ? S_ : 0], dg[q], mu[q]); }
            B200_ADJ_STAGE(1, tsit5_dense_hermite<D>(ulo, du, kf[0], kf[6], c4, a.hHf[0], y))
            B200_ADJ_STAGE(2, tsit5_dense_hermite<D>(ulo, du, kf[0], kf[6], c4, a.hHf[1], y))
            B200_ADJ_STAGE(3, tsit5_dense_hermite<D>(ulo, du, kf[0], kf[6], c4, a.hHf[2], y))
            B200_ADJ_STAGE(4, tsit5_dense_hermite<D>(ulo, du, kf[0], kf[6], c4, a.hHf[3], y))
            B200_ADJ_STAGE(5, _Pragma("unroll") for (int j = 0; j < D; j++) y[j] = ulo[j])
            B200_ADJ_STAGE(6, _Pragma("unroll") for (int j = 0; j < D; j++) y[j] = ulo[j])
#undef B200_ADJ_STAGE
            // ls = lambda(t_n) (row 6 of A is b), ka[6] = FSAL derivative at (t_n, ls, u_n)

#ifdef REV_MIDSYNC
            __syncthreads();
#endif
            if (SA == SA_QUAD) {
                // QuadratureAdjoint: keep the dense reverse solution of this step (adj_sol with save_everystep,
                // src/quadrature_adjoint.jl:527-530): start value (post-jump lambda(t_{n+1})) and the 7 stage derivatives
                R* row = a.adj_dense + (int64_t)n * 8 * cstride + member_gi();
#pragma unroll
                for (int j = 0; j < D; j++) row[(int64_t)j * Npad] = lam[j];
#pragma unroll
                for (int s_ = 0; s_ < 7; s_++)
#pragma unroll
                    for (int j = 0; j < D; j++) row[((int64_t)(1 + s_) * D + j) * Npad] = ka[s_][j];
            }
            if (SA == SA_GK) {
                // GaussKronrodAdjoint on the fixed grid (src/gauss_adjoint.jl:820-825, IntegratingGKSumCallback): error-
                // controlled G3/K7 quadrature of this step, bisected while sum|K - G| >= 1e-7; lam from the adjoint step's own
                // dense output, y from the forward dense output, both at arbitrary theta.  Local time s in [h, 0] above t_n.
                auto node = [&](double sj, double* out) {
                    const R thf = (R)(sj / (double)a.hstep), tha = (R)1 - thf;
                    R wf[7], wa[7], lq[D], yq[D], dgq[P];
#pragma unroll
                    for (int j = 0; j < 7; j++) {
                        wf[j] = a.hstep * (thf * (a.Rpoly[j][0] + thf * (a.Rpoly[j][1] + thf * (a.Rpoly[j][2] + thf * a.Rpoly[j][3]))));
                        wa[j] = a.hstep * (tha * (a.Rpoly[j][0] + tha * (a.Rpoly[j][1] + tha * (a.Rpoly[j][2] + tha * a.Rpoly[j][3]))));
                    }
                    tsit5_dense<D>(lam, ka, wa, lq);
                    tsit5_dense<D>(ulo, kf, wf, yq);
                    Fam::vjp_p(yq, p, lq, dgq);
#pragma unroll
                    for (int q = 0; q < P; q++) out[q] = -(double)dgq[q];
                };
                double accd[P];
#pragma unroll
                for (int q = 0; q < P; q++) accd[q] = 0.0;
                integrate_gk_step<P, 3>(node, (double)a.hstep, 0.0, accd);
#pragma unroll
                for (int q = 0; q < P; q++) mu[q] += (R)accd[q];
            }
            if (SA == SA_GAUSS) {
                // 3-point Gauss-Legendre over this step, pre-jump lambda from the adjoint step's own dense output,
                // y from the forward dense output: dp += (h/2) w_q (df/dp)'(y_q) lam_q  (gauss_adjoint.jl:745-759).
                // Both in Hermite form: lambda at theta_g of the adjoint step (start lam, increment ls - lam, end-point
                // derivatives ka[0], ka[6]) is the point of the y-side row with theta 1 - theta_g = theta_{2-g}, row 6 - g
                R dl[D], cl[D], lq[D];
#pragma unroll
                for (int j = 0; j < D; j++) dl[j] = ls[j] - lam[j];
                tsit5_hermite_c4_du<D>(a.hC4u, ka, cl);
#pragma unroll
                for (int g = 0; g < 3; g++) {
                    tsit5_dense_hermite<D>(lam, dl, ka[0], ka[6], cl, a.hHf[6 - g], lq);
                    tsit5_dense_hermite<D>(ulo, du, kf[0], kf[6], c4, a.hHf[4 + g], y);
                    Fam::vjp_p(y, p, lq, dg);
#pragma unroll
                    for (int q = 0; q < P; q++) mu[q] = fma(tb.hGW[g], dg[q], mu[q]);
                }
            }
#pragma unroll
            for (int j = 0; j < D; j++) { lam[j] = ls[j]; ka[0][j] = ka[6][j]; kf[6][j] = kf[0][j]; }

            // ---- jump at t_n (ReverseLossCallback): lam += dgdu(t_k), FSAL invalidated => recompute ka[0] ----
            const int ks = a.save_of_step[n];
            if (ks >= 0 && !((a.flags & KF_NO_START) && n == 0)) {
                add_cotangent<D, COST>(a, ks, stride, N, member_i(), ulo, lam);
                Fam::vjp_u(ulo, p, lam, ka[0]);
                add_continuous<D, CONT>(a, ulo, ka[0]);
            }
#pragma unroll
            for (int j = 0; j < D; j++) uhi[j] = ulo[j];
            if (EV) {
                const int e = a.event_of_step[n];
                if (e >= 0 && n > 0) { reverse_affect(e, lam, mu, member_i()); need_left = true; }
            }
            if (top && n > 0) {                // hand the group on to the next warp of the ring
                const int lane = (int)(threadIdx.x & 31);
                R* m = s_mig + (size_t)(grp - q4) * NV * 32 + lane;
#pragma unroll
                for (int j = 0; j < D; j++) { m[j * 32] = lam[j]; m[(D + j) * 32] = ka[0][j]; m[(2 * D + j) * 32] = kf[6][j]; m[(3 * D + j) * 32] = uhi[j]; }
#pragma unroll
                for (int q = 0; q < P; q++) m[(4 * D + q) * 32] = mu[q];
                __threadfence_block();
                named_bar_arrive(1 + (grp - q4) * 4 + ((c + 1) & 3), 64);
            }
        }
    }

    gi = member_gi(); active = grp >= 0 && gi < a.N; i = active ? gi : a.N - 1;       // final holder of each group
    if (active) store_state<D>(a.du0, N, i, lam);
    if (a.trace && threadIdx.x == 0) {
        unsigned long long t;
        asm volatile("mov.u64 %0, %%globaltimer;" : "=l"(t));
        a.trace[blockIdx.x * 3 + 2] = t;
    }
    // written out here rather than through store_dp, which reorders this kernel's instructions at the same register count
    if (SHARED_P) {
        if (!active) {
#pragma unroll
            for (int q = 0; q < P; q++) mu[q] = 0.0;
        }
        double mud[P];                         // block / grid reduction in fp64 for both precisions
#pragma unroll
        for (int q = 0; q < P; q++) mud[q] = (double)mu[q];
        reduce_dp<P>(mud, a.partials, a.dp, a.ticket, &a.p2p);
    } else if (active) {
#pragma unroll
        for (int q = 0; q < P; q++) a.dp_members[(int64_t)q * N + i] = mu[q];
    }
}

}  // namespace b200adj
