"""Direct interface: adjoint_sensitivities(sol, alg; t, dgdu_discrete, sensealg, ...) -> (du0, dp).

Mirrors /root/reference/src/sensitivity_interface.jl:373-526 (and the Gauss / Quadrature twins
src/gauss_adjoint.jl:766-870, src/quadrature_adjoint.jl:510-633) for an ensemble solution produced by
`solve(EnsembleProblem, alg, EnsembleB200(); ...)`: same keyword names, same defaults, same return convention
(`du0`, and `dp` as a ROW: shape (1, P) for shared parameters, like the reference's `dp'`,
src/sensitivity_interface.jl:503-507).  For an ensemble `du0` is [d, N]; with per-member parameters `dp` is [P, N].
"""
import numpy as np

from . import _lib
from .problems import (FAMILIES, GENERAL_NOISE_FAMILIES, AdjointSensitivityParameterCompatibilityError, AffineCost, ParamAffine,
                       QuadraticRunningCost)
from .sensitivity_algorithms import (B200Adjoint, BacksolveAdjoint, GaussAdjoint, GaussKronrodAdjoint, InterpolatingAdjoint,
                                     QuadratureAdjoint, isnoisemixing, sensealg_name)

FAM_USER_BASE = 100      # B200ADJ_FAM_USER_BASE: ids of registered plug-in families


def _check_noise_mixing(family, sensealg):
    """A diagonal-noise plug-in SDE family's kernels take g_i to depend on u_i and p only (csrc/family_plugin.inc): the
    noisemixing = true diffusion VJP of the reference (src/derivative_wrappers.jl:1165-1211) is not built for it.  A
    general-noise family accepts either value: its diffusion VJP is always the full one, which is what the reference computes
    with noisemixing = true."""
    if sensealg is None or not isnoisemixing(sensealg) or family in GENERAL_NOISE_FAMILIES:
        return
    if FAMILIES.get(family, (0, 0, 0))[2] and _lib.FAM.get(family, -1) >= FAM_USER_BASE:
        raise NotImplementedError(f"noisemixing = true: the SDE family plug-in {family!r} is built for diagonal noise that does not "
                                  "mix (g_i depends on u_i and p only)")


def _check_general_noise(family, stepper, sensealg):
    """EM + BacksolveAdjoint integrates the reference's Ito-transformed drift f - J_{vec G}' vec G (src/sde_tools.jl:29-66),
    which is the Ito correction only for noise that does not mix: it is not built for a general-noise family."""
    inner = sensealg.inner if isinstance(sensealg, B200Adjoint) else sensealg
    if family in GENERAL_NOISE_FAMILIES and stepper == "em" and isinstance(inner, BacksolveAdjoint):
        raise NotImplementedError(f"EM + BacksolveAdjoint is not built for the general-noise SDE family {family!r}: use EulerHeun "
                                  "or InterpolatingAdjoint")


def _check_params(p):
    """src/sensitivity_interface.jl:438-443"""
    if p is None:
        raise ValueError("Your model does not have parameters, and thus it is impossible to calculate the derivative "
                         "of the solution with respect to the parameters.")
    if hasattr(p, "dtype"):
        if "float" not in str(p.dtype):
            raise AdjointSensitivityParameterCompatibilityError()
        return
    try:
        arr = np.asarray(p)
    except Exception:
        raise AdjointSensitivityParameterCompatibilityError()
    if arr.dtype.kind != "f":
        raise AdjointSensitivityParameterCompatibilityError()


def adjoint_sensitivities(sol, alg=None, *, sensealg=None, t=None, dgdu_discrete=None, dgdp_discrete=None,
                          dgdu_continuous=None, dgdp_continuous=None, g=None, no_start=False,
                          abstol=1.0e-6, reltol=1.0e-3, checkpoints=None, corfunc_analytical=None, callback=None,
                          row_dp=True, **kwargs):
    """dgdu_discrete: an `AffineCost` (evaluated in-kernel) or an array Delta[K, d, N] of cotangents at `t`."""
    if sensealg is None:
        sensealg = InterpolatingAdjoint()          # reference default (src/sensitivity_interface.jl:375)
    inner = sensealg.inner if isinstance(sensealg, B200Adjoint) else sensealg
    if not isinstance(inner, (BacksolveAdjoint, InterpolatingAdjoint, QuadratureAdjoint, GaussAdjoint, GaussKronrodAdjoint)):
        raise TypeError("adjoint_sensitivities: sensealg must be one of the continuous adjoints")
    # events: the forward solution carries them (PresetTimeCallback passed to solve, like the reference's tracked callbacks
    # inside sol.prob.kwargs); a different callback for the reverse pass alone is meaningless
    if callback is not None and getattr(sol.engine, "events", None) is None:
        raise NotImplementedError("pass the PresetTimeCallback to solve(); other callbacks/events are not carried on the "
                                  "B200 path (SURVEY.md App. E): delegate to the reference implementation")
    if getattr(sol.engine, "events", None) is not None and isinstance(inner, QuadratureAdjoint):
        raise NotImplementedError("QuadratureAdjoint does not support callbacks")
    # cost functions are members of the NAMED cost family (the device evaluates them in-kernel): dgdu = a .* u + b,
    # dgdp = c .* p + e.  `g` alone (no dgdu_continuous / dgdp_continuous) has both gradients derived from it, as the
    # reference does by AD (src/derivative_wrappers.jl:1427-1440).
    if g is not None:
        if not isinstance(g, QuadraticRunningCost):
            raise NotImplementedError("g must be a QuadraticRunningCost on the B200 path (named cost families only)")
        if dgdu_continuous is None:
            dgdu_continuous = g
        if dgdp_continuous is None and (g.c is not None or g.e is not None):
            dgdp_continuous = ParamAffine(0.0 if g.c is None else g.c, 0.0 if g.e is None else g.e)
    if dgdu_continuous is not None and not isinstance(dgdu_continuous, QuadraticRunningCost):
        raise NotImplementedError("dgdu_continuous must be a QuadraticRunningCost on the B200 path")
    if dgdp_continuous is None and isinstance(dgdu_continuous, QuadraticRunningCost) and (dgdu_continuous.c is not None or dgdu_continuous.e is not None):
        dgdp_continuous = ParamAffine(0.0 if dgdu_continuous.c is None else dgdu_continuous.c, 0.0 if dgdu_continuous.e is None else dgdu_continuous.e)
    for nm, fn in (("dgdp_discrete", dgdp_discrete), ("dgdp_continuous", dgdp_continuous)):
        if fn is not None and not isinstance(fn, ParamAffine):
            raise NotImplementedError(f"{nm} must be a ParamAffine on the B200 path (named cost families only)")
    if dgdp_continuous is not None and dgdu_continuous is None:
        dgdu_continuous = QuadraticRunningCost(0.0, 0.0)
    if dgdp_discrete is not None and dgdu_discrete is None:
        dgdu_discrete = AffineCost(0.0, 0.0)
    if dgdu_discrete is None and dgdu_continuous is None:
        # src/interpolating_adjoint.jl:321-326
        raise ValueError("Either `dgdu_discrete`, `dgdp_discrete`, `dgdu_continuous`, `dgdp_continuous`, or `g` "
                         "must be specified.")
    _check_params(sol.p)
    eng = sol.engine
    if eng is None:
        raise RuntimeError("solution carries no live device handle")
    _check_noise_mixing(eng.family, sensealg)
    _check_general_noise(eng.family, getattr(sol.alg, "code", None), sensealg)
    ts = sol.t if t is None else np.asarray(t, dtype=np.float64)
    if dgdu_discrete is None:
        ts = np.zeros(0)                                   # continuous cost only: no jumps (discrete = false in the reference)
    name = sensealg_name(inner)
    # Backsolve through the direct interface: checkpoints default to sol.t = every forward step
    # (src/sensitivity_interface.jl:433); pass `checkpoints=ts` for the rrule behaviour.
    every = False
    checkpointing = True
    if isinstance(inner, BacksolveAdjoint):
        checkpointing = inner.checkpointing
        every = checkpoints is None
    cost = dgdu_discrete if isinstance(dgdu_discrete, AffineCost) else None
    if dgdu_discrete is None:
        cost = AffineCost(0.0, 0.0)
    eng.set_reverse(name, cost=cost, no_start=no_start, checkpointing=checkpointing, ckpt_every_step=every, t=ts, dgdp=dgdp_discrete)
    if dgdu_continuous is not None or getattr(eng, "_cont_on", False):
        bc = lambda x, n: None if x is None else np.ascontiguousarray(np.broadcast_to(np.asarray(x, dtype=np.float64), (n,)))
        if dgdu_continuous is None:
            eng.handle.set_continuous_cost(False, 0.0, 0.0)
        else:
            eng.handle.set_cost_family(1, bc(dgdu_continuous.a, eng.d), bc(dgdu_continuous.b, eng.d),
                                       bc(getattr(dgdp_continuous, "c", None), eng.P), bc(getattr(dgdp_continuous, "e", None), eng.P))
        eng._cont_on = dgdu_continuous is not None
    # adjoint solve tolerances are keywords of adjoint_sensitivities (src/sensitivity_interface.jl:432; used by the adaptive
    # steppers only); quadgk tolerances come from the sensealg (src/quadrature_adjoint.jl:517)
    is_quad = isinstance(inner, QuadratureAdjoint)
    if getattr(eng, "adaptive", False) or is_quad:
        eng.handle.set_tolerances(abstol if getattr(eng, "adaptive", False) else 0.0, reltol if getattr(eng, "adaptive", False) else 0.0,
                                  inner.abstol if is_quad else 0.0, inner.reltol if is_quad else 0.0)
    du0, dp = eng.reverse(None if cost is not None else dgdu_discrete)
    from .distributed import allreduce_dp
    dp = allreduce_dp(dp, eng)
    if row_dp and eng.shared_p:
        dp = dp.reshape(1, -1)
    return du0, dp
