"""Problem, algorithm and solution types on the host side.

These mirror the UPSTREAM SciMLBase / OrdinaryDiffEq / StochasticDiffEq objects the reference's hot path is handed
(ODEProblem, SDEProblem, EnsembleProblem, Tsit5(), Rosenbrock23(), EM(), EulerHeun(); SURVEY.md section 1 rows U1/U3),
reduced to what the device path needs.  The RHS is a NAMED family (string) instead of a Julia closure: the device
code for f and its VJPs is hand-written per family (csrc/families.cuh), which is the plug-in seam user-supplied
`ODEFunction(f; vjp, vjp_p)` occupies in the reference (src/derivative_wrappers.jl:284-359).
"""
from dataclasses import dataclass, field
from typing import Any, Callable, Optional, Sequence, Tuple

import numpy as np

FAMILIES = {
    # name: (d, P, m)
    "lv": (2, 4, 0), "lorenz": (3, 3, 0), "robertson": (3, 3, 0), "sde_lv": (2, 6, 2), "sde_linear": (2, 2, 2),
    "ball": (2, 2, 0),           # bouncing ball x' = v, v' = -p[0]; p = [gravity, restitution] (adaptive Tsit5; ContinuousCallback)
    "relax": (1, 2, 0),          # u' = p[0] - u; p = [steady state, injected amount] (test/Callbacks2/continuous_callbacks.jl:317-324)
    "mlp": (2, 4482, 0),         # 2 -> 64 -> 64 -> 2 tanh MLP, p = [W1, b1, W2, b2, W3, b3] column-major flattened
}
# conditions compiled into a registered plug-in family (VectorContinuousCallback); families not listed have none
FAMILY_CONDITIONS = {}


class AdjointSensitivityParameterCompatibilityError(TypeError):
    """src/sensitivity_interface.jl:25-29"""

    def __init__(self):
        super().__init__("Adjoint sensitivity analysis functionality requires being able to solve a differential "
                         "equation defined by the parameter struct `p`: `p` must be a flat floating-point array "
                         "(or None) on the B200 path")


@dataclass
class ODEProblem:
    f: str                       # named RHS family
    u0: Any
    tspan: tuple
    p: Any = None
    callback: Any = None
    mass_matrix: Any = None
    kwargs: dict = field(default_factory=dict)
    is_sde = False


@dataclass
class SDEProblem:
    f: str                       # named drift+diffusion family (diagonal noise)
    u0: Any
    tspan: tuple
    p: Any = None
    callback: Any = None
    seed: int = 0
    noise: Any = None            # explicit Wiener increments dW[S][m][N] (NoiseGrid-like)
    kwargs: dict = field(default_factory=dict)
    is_sde = True


@dataclass
class EnsembleProblem:
    """EnsembleProblem(prob; prob_func).  `prob_func(prob, i)` -> (u0_i, p_i or None) is evaluated on the host to
    materialise u0[d, N] (and optionally p[P, N]) as in test/Core4/ensembles.jl:22-24; alternatively pass the
    arrays directly with `u0s` / `ps`."""
    prob: Any
    prob_func: Optional[Callable] = None
    u0s: Any = None              # [d, N]
    ps: Any = None               # [P, N] per-member parameters (None => shared prob.p)


# ---- solver algorithms ----
@dataclass(frozen=True)
class Tsit5:
    adaptive: bool = False       # False: fixed step dt; True: error-controlled (abstol / reltol keywords of solve)
    dt: float = 0.0

    @property
    def code(self):
        return "tsit5_adaptive" if self.adaptive else "tsit5_fixed"


@dataclass(frozen=True)
class Rosenbrock23:
    code = "rosenbrock23"


@dataclass(frozen=True)
class EM:
    dt: float = 0.0
    code = "em"


@dataclass(frozen=True)
class EulerHeun:
    dt: float = 0.0
    code = "euler_heun"


# ---- ensemble algorithms ----
@dataclass(frozen=True)
class EnsembleB200:
    """Batched device solve of the whole ensemble (the dispatch the reference lacks; SURVEY.md finding 2).
    With torch.distributed initialised the members are sharded contiguously over ranks (one process per GPU)."""
    device: Optional[int] = None
    buffers_on_device: Optional[bool] = None   # None: infer from the input arrays
    presharded: bool = False                   # True: the arrays passed in are already THIS rank's shard (no slicing; dp is
                                               # still all-reduced, Philox member offset = rank * local N)
    pin_outputs: bool = False                  # host-buffer mode: results land in page-locked buffers owned (and reused) by the handle
    reuse_handle: bool = False                 # keep ONE device handle per configuration across solve() calls (the
                                               # previous solution's checkpoints are overwritten by the next solve)


@dataclass
class EnsembleSolution:
    """Result of `solve(EnsembleProblem, alg, EnsembleB200(); ...)`: u[K, d, N] at ts[K] (sensitivity_solution)."""
    prob: Any
    alg: Any
    t: np.ndarray
    u: Any
    retcode: Any = None          # int32[N]: 0 = Success, 1 = Unstable (non-finite)
    dense: bool = True
    engine: Any = None           # live device handle (checkpoints) for the reverse pass
    u0: Any = None
    p: Any = None

    def __len__(self):
        return self.u.shape[-1]


@dataclass(frozen=True)
class AffineCost:
    """dgdu_discrete(out, u, p, t, i) = a .* u .+ b evaluated in-kernel (a, b scalars or one entry per state component);
    `dg(out,u,p,t,i) = out .= u .- 2` (test/Core3/adjoint.jl:1169-1171) is AffineCost(1.0, -2.0), the `out[1] = 2u[1];
    out[2] = 0` of test/Core7/mixed_costs.jl:226-230 is AffineCost([2, 0], 0).  Loss = sum_k sum_j (a_j/2 u_j^2 + b_j u_j)."""
    a: Any = 0.0
    b: Any = 1.0

    @property
    def is_scalar(self):
        return np.ndim(self.a) == 0 and np.ndim(self.b) == 0


@dataclass(frozen=True)
class ParamAffine:
    """dgdp_discrete(out, u, p, t, i) / dgdp_continuous(out, u, p, t) = c .* p .+ e: the parameter part of the named cost
    family (cost term sum_q c_q/2 p_q^2 + e_q p_q).  `out[1] = 1; out[2:4] .= 0` of test/Core7/mixed_costs.jl:50-56, 231-237
    (g = u1^2 + p1) is ParamAffine(0, [1, 0, 0, 0])."""
    c: Any = 0.0
    e: Any = 0.0


@dataclass(frozen=True)
class QuadraticRunningCost:
    """Continuous cost g(u, p, t) = sum_j a_j/2 u_j^2 + b_j u_j (+ sum_q c_q/2 p_q^2 + e_q p_q): dgdu_continuous = a .* u + b,
    dgdp_continuous = c .* p + e, evaluated in-kernel at every adjoint stage (accumulate_cost!,
    src/derivative_wrappers.jl:1411-1442; test/Core7/mixed_costs.jl:19-110).  Pass it as `dgdu_continuous=` (with
    `dgdp_continuous=ParamAffine(c, e)` if the cost depends on p) or alone as `g=` (both gradients derived from it, the
    "without dgdu_continuous, dgdp_continuous" call of mixed_costs.jl:188-196).  Loss contribution = integral of g."""
    a: Any = 0.0
    b: Any = 0.0
    c: Any = None
    e: Any = None


@dataclass(frozen=True)
class ContinuousCallback:
    """ContinuousCallback(condition, affect!) of the named family the device path carries (SURVEY.md 8f rank 2; the
    reference's treatment: src/callback_tracking.jl:232-480, docs/src/examples/hybrid_jump/bouncing_ball.md):
      condition(u, t, integrator) = u[idx] - level      (fires on a zero crossing; direction -1 = downwards only, i.e.
                                                         affect_neg! = nothing ..., +1 upwards only, 0 both)
      affect!(integrator): u .= scale .* u .+ shift, then u[p_comp] = p_sign * p[p_param] * u[p_comp]   (if p_comp is set)
    A parameter-dependent level and an additive parameter affect are part of the family: level + level_coef * p[level_param]
    and u[add_comp] += add_coef * p[add_param] -- "condition = u[1] - 3//4 * p[1]; affect! = u[1] += p[2]"
    (test/Callbacks2/continuous_callbacks.jl:317-345) is ContinuousCallback(idx=0, direction=0, level_param=0, level_coef=0.75,
    add_comp=0, add_param=1, add_coef=1.0).  The non-linear affect of the reference's tests, "integrator.u[2] = integrator.u[2]^2"
    (:222-250), is sq_comp=1 (u[sq_comp] <- sq_coef * u[sq_comp]^2 in place of that component's affine map).
    The bouncing ball "integrator.u[2] = -integrator.p[2] * integrator.u[2]" when u[1] crosses 0 downwards is
    ContinuousCallback(idx=0, direction=-1, p_comp=1, p_param=1, p_sign=-1.0).  Indices are 0-based.
    save_positions = (false, false) only; every ensemble member finds its own event times on the device."""
    idx: int
    level: float = 0.0
    direction: int = -1
    scale: Any = None
    shift: Any = None
    p_comp: Optional[int] = None
    p_param: int = 0
    p_sign: float = 1.0
    max_events: int = 64
    save_positions: Tuple[bool, bool] = (False, False)
    level_param: Optional[int] = None
    level_coef: float = 0.0
    add_comp: Optional[int] = None
    add_param: int = 0
    add_coef: float = 0.0
    sq_comp: Optional[int] = None
    sq_coef: float = 1.0

    def key(self):
        sc = None if self.scale is None else np.asarray(self.scale, dtype=np.float64).tobytes()
        sh = None if self.shift is None else np.asarray(self.shift, dtype=np.float64).tobytes()
        return ("cc", self.idx, self.level, self.direction, sc, sh, self.p_comp, self.p_param, self.p_sign, self.max_events,
                self.level_param, self.level_coef, self.add_comp, self.add_param, self.add_coef, self.sq_comp, self.sq_coef)


@dataclass(frozen=True)
class VectorContinuousCallback:
    """VectorContinuousCallback(condition, affect!, NC) whose condition(out, u, t, integrator) and affect!(integrator, ev) are
    the ones compiled into the problem's family (a plug-in built with has_events=True: csrc/family_plugin.inc,
    examples/vector_callback_families.cuh); with NC = 1 it is a ContinuousCallback with a general condition.  The reference's
    treatment: src/callback_tracking.jl:232-480.
      direction: -1 (a condition fires when it crosses zero downwards only), +1 (upwards only) or 0 (both); a scalar or one
                 entry per condition
      max_events: per-member capacity of the event list (status 3 when exceeded)
    save_positions = (false, false) only; every ensemble member finds its own events on the device, and the conditions whose
    crossings land on the same bits fire together (ev has one non-zero entry per condition that fired)."""
    direction: Any = 0
    max_events: int = 64
    save_positions: Tuple[bool, bool] = (False, False)

    def directions(self, nc):
        d = np.asarray(self.direction, dtype=np.int32).reshape(-1)
        if d.size == 1:
            d = np.full(nc, d[0], dtype=np.int32)
        if d.shape != (nc,):
            raise ValueError(f"VectorContinuousCallback: direction must be a scalar or have {nc} entries")
        return np.ascontiguousarray(d)

    def key(self):
        return ("vcc", np.asarray(self.direction, dtype=np.int32).tobytes(), self.max_events)


def saveat_to_times(saveat, tspan):
    """saveat::Number -> t0:saveat:t1 with the end point appended (src/concrete_solve.jl:718-725, 2827-2831);
    arrays are sorted (:752-756)."""
    t0, t1 = float(tspan[0]), float(tspan[1])
    if np.isscalar(saveat):
        n = int(np.floor((t1 - t0) / saveat * (1 + 1e-12)))
        ts = t0 + saveat * np.arange(n + 1)
        if abs(ts[-1] - t1) > 1e-12 * max(1.0, abs(t1)):
            ts = np.append(ts, t1)
        else:
            ts[-1] = t1
        return ts
    return np.sort(np.asarray(saveat, dtype=np.float64))


# ---- callbacks: the named affect family the device path carries (SURVEY.md 8f rank 2) ---------------------------------
@dataclass(frozen=True)
class AffineAffect:
    """affect!(integrator): integrator.u .= scale .* integrator.u .+ shift  (per component).  "u[1] += 2" is
    AffineAffect(scale=[1, 1], shift=[2, 0]); "u[1] = 2" is AffineAffect(scale=[0, 1], shift=[2, 0])
    (test/Callbacks1/discrete_callbacks.jl:263-293)."""
    scale: Any
    shift: Any
    p_scale: Any = None          # parameter-changing affect integrator.p .= p_scale .* integrator.p .+ p_shift
    p_shift: Any = None          # ("p .= 2p .- 0.5" of discrete_callbacks.jl:294-303 is p_scale=2, p_shift=-0.5)
    # affect that adds a parameter to a state, u[add_comp] += add_coef * p[add_param] (0-based; the "Dosing example"
    # integrator.u[1] += integrator.p[2] of discrete_callbacks.jl:401-427 is add_comp=0, add_param=1, add_coef=1.0)
    add_comp: Optional[int] = None
    add_param: int = 0
    add_coef: float = 1.0


@dataclass(frozen=True)
class PresetTimeCallback:
    """DiffEqCallbacks.PresetTimeCallback(tstops, affect!) / a DiscreteCallback with condition `t in tstops` and those
    tstops passed to solve: the affect fires at the preset times, which become tstops of the forward and reverse solves.
    `affect` is one AffineAffect for every time or a list with one per time.  save_positions = (false, false) is the only
    mode carried on the device (no extra saved points)."""
    tstops: Any
    affect: Any
    save_positions: Tuple[bool, bool] = (False, False)

    def tables(self, d, P=0):
        t = np.asarray(self.tstops, dtype=np.float64).reshape(-1)
        order = np.argsort(t, kind="stable")
        aff = self.affect if isinstance(self.affect, (list, tuple)) else [self.affect] * len(t)
        if len(aff) != len(t):
            raise ValueError("PresetTimeCallback: one affect per time (or a single affect)")
        sc = np.stack([np.broadcast_to(np.asarray(a.scale, dtype=np.float64), (d,)) for a in aff]) if len(t) else np.zeros((0, d))
        sh = np.stack([np.broadcast_to(np.asarray(a.shift, dtype=np.float64), (d,)) for a in aff]) if len(t) else np.zeros((0, d))
        if any(a.p_scale is not None or a.p_shift is not None for a in aff):
            ps = np.stack([np.broadcast_to(np.asarray(1.0 if a.p_scale is None else a.p_scale, dtype=np.float64), (P,)) for a in aff])
            pc = np.stack([np.broadcast_to(np.asarray(0.0 if a.p_shift is None else a.p_shift, dtype=np.float64), (P,)) for a in aff])
            return t[order], sc[order], sh[order], ps[order], pc[order]
        return t[order], sc[order], sh[order]

    def param_shift(self):
        """(comp[E], param[E], coef[E]) in event-time order for b200adj_set_event_param_shift, or None."""
        t = np.asarray(self.tstops, dtype=np.float64).reshape(-1)
        aff = self.affect if isinstance(self.affect, (list, tuple)) else [self.affect] * len(t)
        if not any(a.add_comp is not None for a in aff):
            return None
        order = np.argsort(t, kind="stable")
        comp = np.array([-1 if a.add_comp is None else a.add_comp for a in aff], dtype=np.int32)[order]
        par = np.array([a.add_param for a in aff], dtype=np.int32)[order]
        coef = np.array([a.add_coef for a in aff], dtype=np.float64)[order]
        return comp, par, coef
