/*
 * b200adj.h -- C ABI of libb200adj.so, the Hopper-native (H100, sm_90a) ensemble continuous-adjoint engine.
 *
 * This is the drop-in boundary for ONE hot path of SciML/SciMLSensitivity.jl v7.112.3: the reverse-mode
 * continuous adjoint (InterpolatingAdjoint / GaussAdjoint / QuadratureAdjoint / BacksolveAdjoint) evaluated
 * over an ensemble of independent trajectories.  The reference is pure Julia and has no FFI for this path;
 * the entry points below are what a `ccall` layer binds from a new
 *     SciMLBase._concrete_solve_adjoint(prob, alg, sensealg::B200Adjoint{Inner}, u0, p, originator, args...; kw...)
 * method (shape of /root/reference/src/concrete_solve.jl:523-543,1041 and of the extension precedent
 * ext/SciMLSensitivityMooncakeExt.jl:123-240).  See INTEGRATION.md for the Julia stub.
 *
 * Rules: plain C types only; every call returns int32 (0 = ok, <0 = error, see B200ADJ_ERR_*); no exceptions,
 * no callbacks into the host language, no global mutable state; a handle is single-owner (not thread-safe),
 * one handle per GPU.  The library has NO CPU fallback: b200adj_create fails with B200ADJ_ERR_NO_DEVICE when no
 * CUDA device is usable.
 *
 * Layouts (trajectory-minor SoA, element type per cfg.dtype):
 *   u0[d][N]   p[P] (shared_p=1) or p[P][N]   saved[K][d][N]   dLdu[K][d][N]
 *   du0[d][N]  dp[P] (shared_p=1: summed over the N members of this handle) or dp[P][N]
 *   dW[S][m][N] Wiener increments (SDE steppers), S = round((t1-t0)/dt)
 */
#ifndef B200ADJ_H
#define B200ADJ_H
#include <stdint.h>
#ifdef __cplusplus
extern "C" {
#endif

/* rhs_family: named RHS families whose f, (df/du)'lam and (df/dp)'lam are hand-differentiated device code.
 * Replaces the AD back-ends behind vecjacobian! (src/derivative_wrappers.jl:256-267, :435-1163). */
enum {
    B200ADJ_FAM_LV = 0,         /* Lotka-Volterra d=2 P=4   (test/Core1/concrete_solve_derivatives.jl:106-127) */
    B200ADJ_FAM_LORENZ = 1,     /* Lorenz d=3 P=3           (test/Core3/adjoint.jl:1160-1167)                  */
    B200ADJ_FAM_ROBERTSON = 2,  /* Robertson d=3 P=3        (test/Core2/stiff_adjoints.jl:256-263, 3-param)    */
    B200ADJ_FAM_SDE_LV = 3,     /* LV drift + diag noise g_i = p[4+i] u_i, d=2 P=6 m=2 (Core1/...:737-760)      */
    B200ADJ_FAM_MLP = 4,        /* 2 -> H -> H -> 2 tanh MLP (docs/src/Benchmark.md:49-52), P = H*H+6H+2        */
    B200ADJ_FAM_SDE_LINEAR = 5, /* du_i = p0 u_i dt + p1 u_i dW_i, any d (test/SDE1/sde_stratonovich.jl:22-31)  */
    B200ADJ_FAM_BALL = 6,       /* bouncing ball x' = v, v' = -p0, p = [gravity, restitution], d=2 P=2
                                   (docs/src/examples/hybrid_jump/bouncing_ball.md; adaptive Tsit5 only)          */
    B200ADJ_FAM_RELAX = 7       /* u' = p0 - u, p = [steady state, injected amount], d=1 P=2
                                   (test/Callbacks2/continuous_callbacks.jl:317-324; adaptive Tsit5 only)         */
};
/* User RHS families (SURVEY.md 8f rank 4; replaces the user `ODEFunction(f; vjp, vjp_p, jac, paramjac)` seam of
 * src/derivative_wrappers.jl:284-359, test/Core3/user_vjp.jl:14-38): a family PLUG-IN is a shared library built from a
 * header with one struct of the shape of csrc/families.cuh (see csrc/family_plugin.inc; python -m
 * scimlsensitivity_jl_b200.family_plugin builds it).  Registering it yields a family id for cfg.rhs_family.  F64; fixed-step
 * and adaptive Tsit5 with all sensealgs and events; Rosenbrock23 when the struct also supplies jac / djac / dvjp_p.  A
 * diagonal-noise SDE family (B200ADJ_FAMILY_SDE: drift f, diffusion g and their VJPs) runs on EM / EulerHeun with
 * BacksolveAdjoint / InterpolatingAdjoint, and on no ODE stepper.  So does a general-noise SDE family
 * (B200ADJ_FAMILY_SDE_GENERAL: a D x M diffusion G with 1 <= M <= 4 -- scalar noise M = 1, non-diagonal, non-square, or diagonal
 * noise that mixes), except EM with BacksolveAdjoint. */
#define B200ADJ_FAM_USER_BASE 100
int32_t b200adj_register_family(const char* plugin_path, int32_t* family_id);
int32_t b200adj_family_info(int32_t family_id, int32_t* d, int32_t* P, const char** name);

/* sensealg: which *SensitivityFunction / driver is run (src/sensitivity_algorithms.jl:254-278,378-405,486-510,591-611) */
enum { B200ADJ_SA_INTERPOLATING = 0, B200ADJ_SA_GAUSS = 1, B200ADJ_SA_QUADRATURE = 2, B200ADJ_SA_BACKSOLVE = 3,
       B200ADJ_SA_GAUSSKRONROD = 4 /* GaussKronrodAdjoint (src/sensitivity_algorithms.jl:689-703, src/gauss_adjoint.jl:820-825): adaptive steppers */ };
/* stepper: the `alg` handed to solve() for both the forward and the adjoint problem (src/sensitivity_interface.jl:487-491) */
enum { B200ADJ_ST_TSIT5_FIXED = 0, B200ADJ_ST_ROSENBROCK23 = 1, B200ADJ_ST_EM = 2, B200ADJ_ST_EULER_HEUN = 3,
       B200ADJ_ST_TSIT5_ADAPTIVE = 4 /* error-controlled Tsit5 (PI controller), abstol/reltol; cfg.dt > 0 = initial step */ };
enum { B200ADJ_F64 = 0, B200ADJ_F32 = 1, B200ADJ_BF16_F32ACC = 2 };
/* cost_kind: how the discrete cotangent dgdu_discrete(out,u,p,t,i) is obtained at save time t_k
 * (ReverseLossCallback, src/adjoint_common.jl:754-821).  EXPLICIT = read column k of the array passed to
 * b200adj_reverse (the rrule pullback's Delta, src/concrete_solve.jl:778-947); AFFINE = a*u(t_k)+b evaluated
 * in-kernel (the dg(out,u,p,t,i) = out .= u .- 2 of test/Core3/adjoint.jl:1169-1171 is a=1, b=-2). */
enum { B200ADJ_COST_EXPLICIT = 0, B200ADJ_COST_AFFINE = 1 };

/* flags */
#define B200ADJ_FLAG_NO_START            1u   /* skip the jump at t0 (src/adjoint_common.jl:761)                    */
#define B200ADJ_FLAG_NO_CHECKPOINTING    2u   /* BacksolveAdjoint(checkpointing=false)                              */
#define B200ADJ_FLAG_CKPT_EVERY_STEP     4u   /* Backsolve: checkpoints = sol.t (direct interface default,         */
                                              /* src/sensitivity_interface.jl:433) instead of the save times        */
#define B200ADJ_FLAG_STORED_NOISE        8u   /* SDE: keep dW[S][m][N] in HBM (reference behaviour, reverse(sol.W)) */
                                              /* instead of regenerating it from the Philox counter in reverse      */

#define B200ADJ_FLAG_TRACE              16u   /* record (smid, start, end) of every block of the reverse kernel      */
#define B200ADJ_FLAG_NO_ROTATE          32u   /* tuning: launch exactly block_threads threads, no travelling warp groups */
#define B200ADJ_FLAG_DENSE_FORWARD      64u   /* fixed-step Tsit5: keep the DENSE forward solution (k1..k7 per step, per member) so   */
                                              /* that save / jump times may lie off the dt grid (chosen automatically when cfg.saveat */
                                              /* has off-grid entries; set it to re-target the reverse pass to off-grid times later)  */
#define B200ADJ_FLAG_NCCL_ALLREDUCE    128u   /* multi-GPU: sum dp with ncclAllReduce instead of the all-reduce fused into the reverse    */
                                              /* kernel over peer-memory mailboxes (the default whenever the GPUs can map each other)    */
#define B200ADJ_FLAG_CHECKPOINT_SAVES  256u   /* adaptive Tsit5: checkpointed save intervals (see checkpoint_every below) */
/* flags fixed at create (the others can be changed per reverse pass by b200adj_set_reverse_options) */
#define B200ADJ_CREATE_FLAGS (B200ADJ_FLAG_STORED_NOISE | B200ADJ_FLAG_TRACE | B200ADJ_FLAG_NO_ROTATE | B200ADJ_FLAG_DENSE_FORWARD | B200ADJ_FLAG_NCCL_ALLREDUCE | \
                              B200ADJ_FLAG_CHECKPOINT_SAVES)

/* error codes */
#define B200ADJ_OK                 0
#define B200ADJ_ERR_INVALID       -1   /* null pointer / bad enum / inconsistent sizes                     */
#define B200ADJ_ERR_UNSUPPORTED   -2   /* valid for the reference, not built here: delegate to reference   */
#define B200ADJ_ERR_NO_DEVICE     -3   /* no usable CUDA device (there is no CPU fallback)                 */
#define B200ADJ_ERR_CUDA          -4   /* CUDA runtime error, text in b200adj_last_error                   */
#define B200ADJ_ERR_STATE         -5   /* reverse before forward, etc.                                     */
#define B200ADJ_ERR_OOM           -6

typedef struct b200adj_cfg {
    int32_t rhs_family, sensealg, stepper, dtype;
    int32_t d, P, m, K;
    int64_t N;                       /* ensemble members owned by THIS handle (this GPU's shard)          */
    double  t0, t1, dt;              /* fixed step (ST_TSIT5_FIXED / EM / EULER_HEUN), initial dt hint else */
    double  abstol, reltol;          /* adaptive steppers: forward and adjoint solves                      */
    double  quad_abstol, quad_reltol;/* QuadratureAdjoint quadgk tolerances (src/sensitivity_algorithms.jl:493-503) */
    const double* saveat;            /* K ascending save times (host pointer, copied by create)            */
    int32_t shared_p;                /* 1: one p for all members, dp summed; 0: per-member p and dp        */
    int32_t buffers_on_device;       /* 1: all data pointers passed to forward/reverse are device pointers */
    int32_t device;                  /* CUDA device ordinal                                                */
    int32_t cost_kind;
    double  cost_a, cost_b;
    uint64_t seed;                   /* Philox seed for SDE Wiener increments                              */
    int64_t traj_offset;             /* global index of member 0 (keeps Philox streams shard-independent)  */
    int32_t checkpoint_every;        /* fixed-step Tsit5: keep the forward state every C steps only; the reverse pass re-solves each */
                                     /* C-step segment into shared memory (CheckpointSolution, src/interpolating_adjoint.jl:54-112,  */
                                     /* 206-278; src/gauss_adjoint.jl:57-95, 167-212).  0 or 1 = every step                          */
                                     /* The adaptive Tsit5 stepper checkpoints with B200ADJ_FLAG_CHECKPOINT_SAVES instead: the forward */
                                     /* pass keeps, per member and save interval, only the step state (t_n, u_n, f(u_n), first-attempt */
                                     /* step size, qold) of the step that holds the interval's lower bound; the reverse pass re-solves */
                                     /* one interval at a time and gets the gradient of the full dense solution bit for bit.  The      */
                                     /* intervals are bounded by t0, the save times inside (t0, t1) and t1.  Interpolating / Gauss /   */
                                     /* GaussKronrod, no events or continuous callbacks, and the reverse pass keeps the forward save   */
                                     /* times (everything else is B200ADJ_ERR_UNSUPPORTED).  max_steps then sizes ONE interval.        */
    uint32_t flags;
    int32_t mlp_hidden;              /* FAM_MLP hidden width                                               */
    int32_t block_threads;           /* 0 = library default; tuning knob                                   */
    int32_t max_steps;               /* adaptive steppers: per-member step capacity of the dense forward / reverse solutions */
                                     /* (the reference's maxiters); 0 = 4096.  With B200ADJ_FLAG_CHECKPOINT_SAVES: the accepted */
                                     /* steps of ONE save interval (pass the longest interval's count); a member that needs more */
                                     /* gets status 2 and NaN gradients, the total is bounded by the iteration cap only          */
    int32_t reserved0;               /* must be 0                                                          */
} b200adj_cfg;

/* create: validates cfg, allocates checkpoints/partials on cfg.device, uploads tableaux.  Replaces the set-up done
 * by ODEAdjointProblem / SDEAdjointProblem + adjointdiffcache (src/interpolating_adjoint.jl:307-451,
 * src/gauss_adjoint.jl:275-423, src/quadrature_adjoint.jl:93-214, src/backsolve_adjoint.jl:123-419,
 * src/adjoint_common.jl:42-469). */
int32_t b200adj_create(const b200adj_cfg* cfg, void** handle);

/* forward: batched forward solve of all members, keeps per-step checkpoints in HBM, writes the primal at saveat.
 * Replaces the forward solve + sol(ts) of src/concrete_solve.jl:689-770.  saved may be NULL; status[N] (int32,
 * 0 = ok, 1 = non-finite state, 2 = step capacity (cfg.max_steps) exhausted, 3 = more state-dependent events than
 * max_events) may be NULL.  dW_in (SDE only, may be NULL): use these increments instead of Philox. */
int32_t b200adj_forward(void* handle, const void* u0, const void* p, const void* dW_in, void* saved, int32_t* status);

/* reverse: the fused reverse pass (adjoint RHS + VJPs + quadrature + RK update + jumps, all members), then the
 * deterministic reduction of dp.  Replaces _adjoint_sensitivities (src/sensitivity_interface.jl:426-526,
 * src/gauss_adjoint.jl:766-870, src/quadrature_adjoint.jl:510-633) and everything it calls per stage
 * (sense functors, split_states, vecjacobian!, vec_pjac!, ReverseLossCallback).  dLdu may be NULL when
 * cfg.cost_kind != EXPLICIT. */
int32_t b200adj_reverse(void* handle, const void* dLdu, void* du0, void* dp);

/* Change what the NEXT reverse pass computes without redoing the forward pass (checkpoints are sensealg-agnostic):
 * the reference's adjoint_sensitivities(sol, alg; t, dgdu_discrete, sensealg, no_start, checkpoints) takes these per
 * call on an existing `sol` (src/sensitivity_interface.jl:373-526).  K < 0 keeps the current save times. */
int32_t b200adj_set_reverse_options(void* handle, int32_t sensealg, int32_t cost_kind, double cost_a, double cost_b,
                                    uint32_t flags, int32_t K, const double* t);

/* Tolerances of the NEXT reverse pass on an adaptive handle: the adjoint solve's abstol/reltol (the reference takes them
 * as keywords of adjoint_sensitivities, src/sensitivity_interface.jl:432; default = the forward solve's) and the quadgk
 * tolerances of QuadratureAdjoint (sensealg.abstol/.reltol, src/quadrature_adjoint.jl:517).  Values <= 0 keep the current. */
int32_t b200adj_set_tolerances(void* handle, double adj_abstol, double adj_reltol, double quad_abstol, double quad_reltol);

/* Continuous cost functional (dgdu_continuous / dgdp_continuous of adjoint_sensitivities; accumulate_cost!,
 * src/derivative_wrappers.jl:1411-1442): named family g(u) = a/2 |u|^2 + b sum(u), i.e. dgdu_continuous = a u + b,
 * dgdp_continuous = 0, added to the adjoint RHS of the NEXT reverse pass (on top of the discrete cost, if any).
 * Built for the Tsit5 paths (fixed step: all four sensealgs; adaptive: + GaussKronrod); enabled = 0 switches it off.
 * Per-component coefficients and dgdp_continuous: b200adj_set_cost_family(which = 1). */
int32_t b200adj_set_continuous_cost(void* handle, int32_t enabled, double a, double b);

/* Per-component coefficients of the named cost family and its PARAMETER part (dgdp_discrete / dgdp_continuous / g of
 * adjoint_sensitivities, src/sensitivity_interface.jl:373-526; test/Core7/mixed_costs.jl:19-330 uses g = u1^2 + p1, i.e.
 * a = [2, 0], e = [1, 0, 0, 0]):
 *   which = 0, discrete:   l(u, p) = sum_j a_j/2 u_j^2 + b_j u_j + sum_q c_q/2 p_q^2 + e_q p_q  at every save time
 *                          dgdu_discrete = a .* u + b (needs cost_kind = AFFINE), dgdp_discrete = c .* p + e
 *   which = 1, continuous: the same expression as running cost g(u, p) (enables it like b200adj_set_continuous_cost)
 * a, b: [d] or NULL (keep the current, e.g. the scalars of cfg / set_reverse_options); c, e: [P] or NULL (zero).  Host
 * pointers.  The parameter part is built for P <= 8 and is reset by b200adj_set_reverse_options / b200adj_set_continuous_cost
 * (call this after them).  Per save time the discrete dgdp joins the gradient exactly where the reference's
 * ReverseLossCallback adds it (src/adjoint_common.jl:771-783; QuadratureAdjoint: src/quadrature_adjoint.jl:547-553). */
int32_t b200adj_set_cost_family(void* handle, int32_t which, const double* a, const double* b, const double* c, const double* e);

/* Preset-time events of the hybrid system (DiscreteCallback / PresetTimeCallback of the reference with
 * save_positions = (false, false); reverse-pass treatment of src/callback_tracking.jl:232-480): at each times[e] the state
 * of every member becomes u <- scale[e][:] .* u + shift[e][:] ("u[1] += 2", "u[1] = 2" of
 * test/Callbacks1/discrete_callbacks.jl:263-293 are (1, 2) and (0, 2)).  The event times become tstops of the forward and
 * of the reverse solve; the reverse pass applies lam(tau-) = scale .* lam(tau+) after the loss jump of the same time (a
 * save time that coincides with an event records the post-event state).  times ascending, strictly inside (t0, t1);
 * host pointers; E = 0 removes the events.  pscale / pshift [E][P] (both NULL = none): parameter-changing affect
 * p <- pscale[e][:] .* p + pshift[e][:] at the same times (integrator.p .= 2 .* integrator.p .- 0.5, :294-303; the reverse
 * pass scales the accumulated dG/dp by pscale and continues with the pre-event parameters -- reset_p,
 * src/interpolating_adjoint.jl:748-823).  Built for the adaptive Tsit5 stepper with Interpolating / Gauss / Backsolve
 * (the reference's QuadratureAdjoint has no callback support either); call before b200adj_forward. */
int32_t b200adj_set_events(void* handle, int32_t E, const double* times, const double* scale, const double* shift,
                           const double* pscale, const double* pshift);

/* Affect that ADDS A PARAMETER to a state at the preset times above (the reference's "Dosing example",
 * test/Callbacks1/discrete_callbacks.jl:401-427: affect(integrator) = integrator.u[1] += integrator.p[2]): after the affine
 * part of event e, u[comp[e]] += coef[e] * p[param[e]] with the parameters in force before the event (comp[e] < 0: none for
 * that event).  Reverse pass: dG/dp[param[e]] += coef[e] * lam(t_e+)[comp[e]].  Host arrays of length E (the E of the last
 * b200adj_set_events, which also resets this); comp = NULL removes the shifts.  Built on the per-member dense framework
 * (adaptive Tsit5; fixed-step Tsit5 with B200ADJ_FLAG_DENSE_FORWARD). */
int32_t b200adj_set_event_param_shift(void* handle, const int32_t* comp, const int32_t* param, const double* coef);

/* State-dependent event of the hybrid system (ContinuousCallback of the reference; reverse-pass treatment with the implicit
 * event-time correction of src/callback_tracking.jl:232-480; docs/src/examples/hybrid_jump/bouncing_ball.md,
 * test/Callbacks1/continuous_callbacks.jl): condition(u) = u[idx] - level, fired when it crosses zero in `direction`
 * (-1: from positive to non-positive only -- affect_neg! = nothing --, +1: upwards only, 0: both); the affect is of the named
 * affine family u <- scale .* u + shift (NULL = 1 / 0), followed, when pcomp >= 0, by u[pcomp] <- psign * p[pparam] * u[pcomp]
 * ("v = -p[2] * v": pcomp = 1, pparam = 1, psign = -1), save_positions = (false, false).  Each member finds its OWN event
 * times: the forward kernel samples the condition on the dense output of every accepted step (interp_points = 10), bisects
 * the crossing to the last bit and re-takes the step up to it; the reverse kernel uses the member's event list as tstops and
 * applies  lam- = A'lam+ - e_idx [(A f(u-) - f(u+))'lam+] / f(u-)[idx],  dG/dp[pparam] += psign u-[pcomp] lam+[pcomp].
 * Adaptive Tsit5, Interpolating / Gauss / GaussKronrod / Backsolve (QuadratureAdjoint has no callback support in the
 * reference either); not together with b200adj_set_events.  max_events = per-member capacity of the event list (status 3
 * when exceeded).  enabled = 0 removes the callback.  Call before b200adj_forward. */
int32_t b200adj_set_continuous_callback(void* handle, int32_t enabled, int32_t idx, double level, int32_t direction,
                                        const double* scale, const double* shift, int32_t pcomp, int32_t pparam, double psign,
                                        int32_t max_events);
/* Parameter-dependent condition and additive parameter affect of the callback above (the reference's
 * test/Callbacks2/continuous_callbacks.jl:317-345: condition(u,t,integrator) = u[1] - 3//4 * integrator.p[1],
 * affect!(integrator) = integrator.u[1] += integrator.p[2]):  condition = u[idx] - (level + lcoef * p[lparam])  (lparam < 0:
 * none) and, after the affine part of the affect, u[acomp] += acoef * p[aparam]  (acomp < 0: none).  Reverse pass, with
 * w = (A f(u-) - f(u+))'lam+:  dG/dp[lparam] += lcoef * w / f(u-)[idx]  (the event time moves with the level) and
 * dG/dp[aparam] += acoef * lam+[acomp].  qcomp >= 0: the NON-LINEAR affect of the reference's tests, u[qcomp] <- qcoef *
 * u[qcomp]^2 ("integrator.u[2] = integrator.u[2]^2", test/Callbacks2/continuous_callbacks.jl:222-250) in place of that
 * component's affine map; the reverse pass uses its Jacobian 2 qcoef u-[qcomp] where the affine family has `scale`.
 * Call after b200adj_set_continuous_callback (which resets all three to none). */
int32_t b200adj_set_continuous_callback_params(void* handle, int32_t lparam, double lcoef, int32_t acomp, int32_t aparam, double acoef,
                                               int32_t qcomp, double qcoef);
/* event lists found by the last forward pass: counts[N] (host, may be NULL), times[max_events][N] (host, may be NULL) */
int32_t b200adj_event_times(void* handle, int32_t* counts, double* times);

/* Number of conditions compiled into a family (its plug-in was built with B200ADJ_FAMILY_HAS_EVENTS, csrc/family_plugin.inc):
 * the `len` of VectorContinuousCallback(condition, affect!, len).  0 for every built-in family and for plug-ins without events. */
int32_t b200adj_family_conditions(int32_t family, int32_t* nc);
/* Number of Wiener processes of a family (the m of the SDE steppers EM / EulerHeun; m = d for diagonal noise): 2 for the
 * built-in SDE_LV / SDE_LINEAR, M for a plug-in built with B200ADJ_FAMILY_SDE or B200ADJ_FAMILY_SDE_GENERAL
 * (csrc/family_plugin.inc), 0 for every ODE family.  B200ADJ_ERR_INVALID for an unknown family id. */
int32_t b200adj_family_noise(int32_t family, int32_t* m);
/* The shape of a family's noise term (the reference's noise_rate_prototype):
 *   B200ADJ_NOISE_NONE      an ODE family
 *   B200ADJ_NOISE_DIAGONAL  du = f dt + g .* dW, m = d, g_i a function of u_i and p (the built-in SDE_LV / SDE_LINEAR and the
 *                           plug-ins built with B200ADJ_FAMILY_SDE; noisemixing = false)
 *   B200ADJ_NOISE_GENERAL   du = f dt + G dW with G of size d x m (plug-ins built with B200ADJ_FAMILY_SDE_GENERAL); the
 *                           diffusion VJP is the full one of noisemixing = true.  EM + BacksolveAdjoint is UNSUPPORTED: the
 *                           reference's Ito-transformed drift (src/sde_tools.jl:29-66) is not the Ito correction of a noise
 *                           that mixes.
 * B200ADJ_ERR_INVALID for an unknown family id. */
enum { B200ADJ_NOISE_NONE = 0, B200ADJ_NOISE_DIAGONAL = 1, B200ADJ_NOISE_GENERAL = 2 };
int32_t b200adj_family_noise_kind(int32_t family, int32_t* kind);
/* VectorContinuousCallback of the reference (the callback type of test/Callbacks2/vector_continuous_callbacks.jl; reverse-pass
 * treatment of src/callback_tracking.jl:232-480) with the condition(out, u, t, integrator) and affect!(integrator, ev) compiled
 * into the family struct, save_positions = (false, false).  A mode of the continuous callback above: each member finds its own
 * events (all nc conditions are sampled on the dense output of every accepted step, the first crossing interval is bisected to
 * the last bit, conditions whose roots have the same bits fire together), b200adj_event_times reports them and
 * b200adj_event_flags which conditions fired.  The reverse pass applies, with c = the lowest condition that fired,
 *   lam- = mu_u - dg_c/du (w / den),  dG/dp += mu_p - dg_c/dp (w / den),  den = dg_c/du . f(u-) + dg_c/dt,
 *   w = mu_u . f(u-) - lam+ . f(u+),  (mu_u, mu_p) = the affect's VJP with lam+.
 * direction[nc]: -1 downwards only, +1 upwards only, 0 both.  Adaptive Tsit5, Interpolating / Gauss / GaussKronrod / Backsolve;
 * not together with b200adj_set_events; nc must be the family's.  enabled = 0 removes the callback (either mode).  Call before
 * b200adj_forward. */
int32_t b200adj_set_family_events(void* handle, int32_t enabled, int32_t nc, const int32_t* direction, int32_t max_events);
/* event words of the last forward pass with family events: ev[max_events][N] (host); the word of event e of member i has bit 2c
 * set when condition c fired and bit 2c + 1 when it crossed upwards.  Entries past the member's event count are undefined. */
int32_t b200adj_event_flags(void* handle, int32_t* ev);

/* SDE helper for parity tests: copy out the Wiener increments the forward pass used, dW[S][m][N]. */
int32_t b200adj_get_noise(void* handle, void* dW_out);

/* run on a caller-owned CUDA stream (cudaStream_t passed as void*; NULL = the handle's private non-blocking stream;
 * pass cudaStreamLegacy (0x1) for the legacy default stream).  With buffers_on_device=1 every call is asynchronous on
 * that stream; with host buffers forward/reverse return after their D2H copies completed. */
int32_t b200adj_set_stream(void* handle, void* cuda_stream);
/* block until all work queued by this handle has finished */
int32_t b200adj_synchronize(void* handle);
/* number of kernels this handle has launched so far (bench.py's gpu_launches) */
int64_t b200adj_launch_count(void* handle);
/* device memory the handle owns at the time of the call, in bytes (every buffer it allocated and has not freed yet: dense
 * solutions or checkpoints, save tables, staging, lazily allocated QuadratureAdjoint and event buffers).  For an adaptive
 * Tsit5 handle with buffers_on_device = 1 and no events:
 *   N (MS+1) (8 d + 5) 8  +  12 N  +  2 max(K,1) 8  +  max(qgrid+1, ceil(N/32)) P 8  +  4
 *   [+ N n_seg (2 d + 4) 8 with B200ADJ_FLAG_CHECKPOINT_SAVES, n_seg = 1 + the save times inside (t0, t1)]
 * with MS = max_steps (0: 4096) and qgrid = min(ceil(N / 4), 6 n_SM).  Sizes ensembles before they run out of memory. */
int32_t b200adj_device_bytes(void* handle, int64_t* bytes);
/* adaptive steppers: per-member accepted step counts of the last forward / reverse solves (device or host per cfg) */
int32_t b200adj_get_step_counts(void* handle, int32_t* fwd_steps, int32_t* rev_steps);

/* tracing (needs B200ADJ_FLAG_TRACE at create): out[nblocks][3] = (SM id, %globaltimer ns at block start, at block end)
 * of the last reverse launch; call with out = NULL to query nblocks.  Host pointer always. */
int32_t b200adj_get_block_trace(void* handle, uint64_t* out, int32_t* nblocks);

/* ---- multi-GPU (SURVEY.md 8b "multi-GPU handle owns ... one NCCL communicator", 8e) ----
 * One handle per GPU (one process per GPU, or several handles in one process); each handle owns cfg.N members of the
 * ensemble (cfg.traj_offset = global index of its first member).  Rank 0 obtains a 128-byte id, the host broadcasts it over
 * its own channel (Distributed.jl / MPI / a file), every rank attaches its handle.  From then on b200adj_reverse sums dp over
 * the ranks whenever shared_p = 1: the single collective of the path.  When the GPUs can map each other's memory (CUDA IPC /
 * peer access over NVLink) the sum is FUSED into the fixed-step reverse kernel: its last block stores its dp into a mailbox
 * in every peer's HBM, publishes an epoch flag, waits for the peers' flags and adds the slots in rank order -- no collective
 * launch at all (csrc/ode_tsit5.cuh::reduce_dp, csrc/comm.cu).  Otherwise, and for the other steppers, ncclAllReduce on the
 * handle's stream before the D2H copy.  du0 and per-member dp stay sharded.  NCCL is bound with dlopen at the first call; without a usable libnccl.so.2
 * these return B200ADJ_ERR_UNSUPPORTED and single-GPU use is unaffected. */
int32_t b200adj_comm_unique_id(void* id_out /* 128 bytes */);
int32_t b200adj_comm_init(void* handle, int32_t nranks, int32_t rank, const void* unique_id /* 128 bytes; NULL if nranks == 1 */);
/* single-process host driving several GPUs: handles[0..n-1] (one per device) become ranks 0..n-1 of one communicator (the
 * ncclCommInitRank calls are grouped, so one thread may issue this).  The per-gradient b200adj_reverse calls of the n handles
 * must then be issued concurrently (one host thread per handle, e.g. Threads.@threads), as for any NCCL collective. */
int32_t b200adj_comm_init_all(void** handles, int32_t n);
/* in-place sum of `count` reals (cfg.dtype's ABI element type) over the ranks, on the handle's stream; device pointer */
int32_t b200adj_comm_allreduce(void* handle, void* buf, int64_t count);
int32_t b200adj_comm_size(void* handle, int32_t* nranks, int32_t* rank);
/* 1 when the peer mailboxes are mapped and the fixed-step reverse kernel reduces dp itself (no collective launch), else 0 */
int32_t b200adj_comm_is_fused(void* handle);

int32_t b200adj_destroy(void* handle);
const char* b200adj_last_error(void* handle);   /* handle may be NULL: last create() error of this thread */
uint32_t b200adj_version(void);                 /* 0xMMmmpp */
uint32_t b200adj_sizeof_cfg(void);              /* sizeof(b200adj_cfg): lets a binding verify its struct mirror */

#ifdef __cplusplus
}
#endif
#endif
