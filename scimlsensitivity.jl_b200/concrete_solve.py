"""The drop-in seam: `solve(EnsembleProblem, alg, EnsembleB200(); ...)` and `_concrete_solve_adjoint(...)`.

Mirrors /root/reference/src/concrete_solve.jl:523-1042 (the `_concrete_solve_adjoint` method for the continuous
adjoints): forward solve (:689-707), primal output at `saveat` (:713-770), pullback closure (:776-1040) that
scatters the cotangent into the jump buffer (:778-947), calls `adjoint_sensitivities` (:955-976), reshapes `du0`
(:978) and `dp'` (:980-986) and returns the tangent tuple whose arity depends on the AD originator (:1027-1039).
The ensemble dispatch itself does not exist in the reference (SURVEY.md finding 2): there every member goes through
this rrule separately and the outer AD sums the gradients; here all members run in one batched device pass.
"""
import numpy as np

from . import distributed
from .engine import DeviceEnsemble, _is_torch
from .problems import (EM, AffineCost, ContinuousCallback, VectorContinuousCallback, PresetTimeCallback, EnsembleB200, EnsembleProblem, EnsembleSolution, EulerHeun, FAMILIES, GENERAL_NOISE_FAMILIES, ODEProblem,
                       Rosenbrock23, SDEProblem, Tsit5, saveat_to_times)
from .sensitivity_algorithms import (B200Adjoint, BacksolveAdjoint, GaussAdjoint, GaussKronrodAdjoint, InterpolatingAdjoint,
                                     QuadratureAdjoint, sensealg_name)
from .sensitivity_interface import _check_general_noise, _check_noise_mixing, _check_params, adjoint_sensitivities


class NoTangent:
    """ChainRulesCore.NoTangent()"""

    def __repr__(self):
        return "NoTangent()"


class ChainRulesOriginator:   # SciMLBase.ChainRulesOriginator / Enzyme / Mooncake originators (:363-389)
    pass


class TrackerOriginator:      # Tracker / ReverseDiff originators return one fewer leading NoTangent (:1027-1039)
    pass


ReverseDiffOriginator = TrackerOriginator


def _materialise(eprob, trajectories):
    """prob_func on the host -> u0[d, N], p[P] or p[P, N] (test/Core4/ensembles.jl:22-24)."""
    prob = eprob.prob
    if eprob.u0s is not None:
        u0s = eprob.u0s
        ps = eprob.ps
    elif eprob.prob_func is not None:
        cols, pcols = [], []
        for i in range(trajectories):
            out = eprob.prob_func(prob, i)
            u0_i, p_i = out if isinstance(out, tuple) else (out, None)
            cols.append(np.asarray(u0_i, dtype=np.float64).reshape(-1))
            if p_i is not None:
                pcols.append(np.asarray(p_i, dtype=np.float64).reshape(-1))
        u0s = np.stack(cols, axis=1)
        ps = np.stack(pcols, axis=1) if pcols else None
    else:
        u0s = np.repeat(np.asarray(prob.u0, dtype=np.float64).reshape(-1, 1), trajectories, axis=1)
        ps = None
    return u0s, ps


def _check_noise_rate_prototype(prob, d, m):
    """SDEProblem(...; noise_rate_prototype): only a general-noise family takes one, of its own shape (d, m)"""
    proto = getattr(prob, "noise_rate_prototype", None)
    if proto is None:
        return
    if prob.f not in GENERAL_NOISE_FAMILIES:
        raise ValueError(f"noise_rate_prototype: {prob.f!r} is not a general-noise SDE family (build it with noise=\"general\")")
    if tuple(np.shape(proto)) != (d, m):
        raise ValueError(f"noise_rate_prototype has shape {tuple(np.shape(proto))}; the family {prob.f!r} has a ({d}, {m}) diffusion")


def _step_size(alg, kwargs):
    dt = kwargs.get("dt", getattr(alg, "dt", 0.0))
    if isinstance(alg, Rosenbrock23) or (isinstance(alg, Tsit5) and alg.adaptive):
        return float(dt or 0.0)                     # adaptive: error-controlled steps (abstol / reltol keywords); dt = initial step hint
    if not dt or dt <= 0:
        raise ValueError("fixed-step solve needs dt > 0")
    return float(dt)


_HANDLE_CACHE = {}


def clear_handle_cache():
    """Destroy the device handles kept by `EnsembleB200(reuse_handle=True)` solves."""
    for eng in list(_HANDLE_CACHE.values()):
        eng.close()
    _HANDLE_CACHE.clear()


def solve(eprob, alg, ensemblealg=None, *, trajectories=None, saveat=None, sensealg=None, save_start=True,
          save_end=True, save_on=True, u0=None, p=None, _rrule=False, **kwargs):
    """Batched forward solve of an EnsembleProblem on the device; keeps the checkpoints for a later adjoint.
    `_rrule=True` (set by _concrete_solve_adjoint): output times follow the reference's rrule, not the plain solver --
    for the non-Backsolve adjoints save_start / save_end only drop end points when `saveat` is empty; with a number or an
    array the output keeps t0 / t1 and `no_start` ignores the cotangent at t0 instead (src/concrete_solve.jl:713-770, 962)."""
    if not isinstance(eprob, EnsembleProblem):
        eprob = EnsembleProblem(eprob)
    ensemblealg = ensemblealg or EnsembleB200()
    prob = eprob.prob
    callback = kwargs.pop("callback", None) or prob.callback
    ccb = None
    if isinstance(callback, (ContinuousCallback, VectorContinuousCallback)):
        # state-dependent event -- the named condition / affect family, or the conditions and affect compiled into the problem's
        # family: adaptive Tsit5, every member finds its own event times
        kind = type(callback).__name__
        if tuple(callback.save_positions) != (False, False):
            raise NotImplementedError(f"{kind}: save_positions = (false, false) only")
        if not (isinstance(alg, Tsit5) and alg.code == "tsit5_adaptive"):
            raise NotImplementedError(f"{kind}: built for the adaptive Tsit5 stepper")
        ccb, callback = callback, None
    if callback is not None:
        # preset-time affine affects on the Tsit5 steppers
        if not isinstance(callback, PresetTimeCallback):
            raise NotImplementedError("callbacks: PresetTimeCallback(tstops, AffineAffect) and ContinuousCallback(idx, ...) are carried on "
                                      "the B200 path (SURVEY.md App. E); delegate other callbacks to the reference implementation")
        if tuple(callback.save_positions) != (False, False):
            raise NotImplementedError("PresetTimeCallback: save_positions = (false, false) only")
        if not isinstance(alg, Tsit5):
            raise NotImplementedError("PresetTimeCallback: built for the Tsit5 steppers (adaptive, or fixed step with event times on the dt grid)")
    kwargs.pop("tstops", None)                     # the callback's own times are the tstops
    if getattr(prob, "mass_matrix", None) is not None:
        raise NotImplementedError("mass matrices / DAEs are not supported on the B200 path")
    if prob.f not in FAMILIES:
        raise KeyError(f"unknown RHS family {prob.f!r}; known: {sorted(FAMILIES)}")
    d, P, m = FAMILIES[prob.f]
    _check_noise_mixing(prob.f, sensealg)
    _check_general_noise(prob.f, alg.code, sensealg)
    _check_noise_rate_prototype(prob, d, m)
    if u0 is None or p is None:
        if trajectories is None:
            trajectories = eprob.u0s.shape[1] if eprob.u0s is not None else 1
        u0s, ps = _materialise(eprob, trajectories)
        u0 = u0 if u0 is not None else u0s
        if p is None:
            p = ps if ps is not None else prob.p
    _check_params(p)
    N_global = u0.shape[1]
    shared_p = (np.ndim(p) == 1) if not _is_torch(p) else (p.dim() == 1)
    if saveat is None and (isinstance(alg, Rosenbrock23) or (isinstance(alg, Tsit5) and alg.adaptive)):
        raise ValueError("adaptive solve on the B200 path needs explicit saveat times")
    ts = saveat_to_times(saveat if saveat is not None else _step_size(alg, kwargs), prob.tspan)
    _inner = sensealg.inner if isinstance(sensealg, B200Adjoint) else sensealg
    if not _rrule or saveat is None or isinstance(_inner, BacksolveAdjoint):
        if not save_start and len(ts) and ts[0] == prob.tspan[0]:
            ts = ts[1:]
        if not save_end and len(ts) and ts[-1] == prob.tspan[1]:
            ts = ts[:-1]
    on_device = ensemblealg.buffers_on_device if ensemblealg.buffers_on_device is not None else _is_torch(u0)
    rank, world = distributed.world()
    if ensemblealg.presharded:
        lo, hi = rank * N_global, (rank + 1) * N_global          # the inputs are this rank's shard already
    else:
        lo, hi = distributed.shard_bounds(N_global)
        if world > 1:
            u0 = u0[:, lo:hi]
            if not shared_p:
                p = p[:, lo:hi]
    device = ensemblealg.device
    if device is None:
        if _is_torch(u0) and u0.is_cuda:
            device = u0.device.index
        else:
            import os
            device = int(os.environ.get("LOCAL_RANK", "0"))
    inner = sensealg.inner if isinstance(sensealg, B200Adjoint) else (sensealg or InterpolatingAdjoint())
    block = getattr(sensealg, "block_threads", 0) if isinstance(sensealg, B200Adjoint) else 0
    stored = getattr(sensealg, "stored_noise", False) if isinstance(sensealg, B200Adjoint) else False
    ckpt_every = getattr(sensealg, "checkpoint_every", 1) if isinstance(sensealg, B200Adjoint) else 1
    ckpt_saves = bool(getattr(sensealg, "checkpoint_saves", False)) if isinstance(sensealg, B200Adjoint) else False
    ev = callback.tables(d, P) if callback is not None else None
    evp = callback.param_shift() if callback is not None else None
    key = (prob.f, alg.code, hi - lo, ts.tobytes(), tuple(prob.tspan), _step_size(alg, kwargs), shared_p, on_device, device,
           getattr(prob, "seed", 0), lo, block, stored, ckpt_every, kwargs.get("abstol", 1e-6), kwargs.get("reltol", 1e-3),
           None if ev is None else tuple(x.tobytes() for x in ev), None if evp is None else tuple(x.tobytes() for x in evp),
           None if ccb is None else ccb.key(), ckpt_saves)
    eng = _HANDLE_CACHE.get(key) if ensemblealg.reuse_handle else None
    if eng is None:
        eng = DeviceEnsemble(prob.f, sensealg_name(inner), alg.code, hi - lo, ts, prob.tspan, _step_size(alg, kwargs),
                             shared_p=shared_p, on_device=on_device, device=device,
                             seed=getattr(prob, "seed", 0), traj_offset=lo, block_threads=block, stored_noise=stored,
                             quad_abstol=getattr(inner, "abstol", 1e-6), quad_reltol=getattr(inner, "reltol", 1e-3),
                             abstol=kwargs.get("abstol", 1e-6), reltol=kwargs.get("reltol", 1e-3),
                             max_steps=kwargs.get("maxiters", 0), pin_outputs=ensemblealg.pin_outputs,
                             checkpoint_every=ckpt_every, checkpoint_saves=ckpt_saves)
        if ev is not None:
            eng.set_events(*ev)
            if evp is not None:
                eng.set_event_param_shift(*evp)
        if ccb is not None:
            eng.set_continuous_callback(ccb)
        if world > 1 and shared_p:
            distributed.attach_comm(eng)           # the one all-reduce of dp then runs inside b200adj_reverse (csrc/comm.cu)
        if ensemblealg.reuse_handle:
            _HANDLE_CACHE[key] = eng
    dW = getattr(prob, "noise", None)
    if dW is not None and world > 1 and not ensemblealg.presharded:
        dW = dW[:, :, lo:hi]
    saved, status = eng.forward(u0, p, dW=dW, want_saved=save_on)
    return EnsembleSolution(prob=eprob, alg=alg, t=ts, u=saved, retcode=status, dense=True, engine=eng, u0=u0, p=p)


def _concrete_solve_adjoint(prob, alg, sensealg, u0, p, originator=None, *args, save_start=True, save_end=True,
                            saveat=None, save_idxs=None, ensemblealg=None, **kwargs):
    """-> (out, pullback).  `sensealg` is B200Adjoint(inner) (or a bare continuous adjoint)."""
    inner = sensealg.inner if isinstance(sensealg, B200Adjoint) else sensealg
    if not isinstance(inner, (BacksolveAdjoint, InterpolatingAdjoint, QuadratureAdjoint, GaussAdjoint, GaussKronrodAdjoint)):
        raise TypeError("_concrete_solve_adjoint(B200 path): continuous adjoints only")
    _check_params(p)                                                   # :544-549
    eprob = prob if isinstance(prob, EnsembleProblem) else EnsembleProblem(prob)
    d = FAMILIES[eprob.prob.f][0]
    u0_shape = tuple(u0.shape)
    u0m = u0.reshape(d, -1)                                            # u0 any shape -> vec (:978)
    sol = solve(eprob, alg, ensemblealg or EnsembleB200(), saveat=saveat, sensealg=sensealg, save_start=save_start,
                save_end=save_end, u0=u0m, p=p, _rrule=True, **kwargs)
    ts = sol.t
    only_end = len(ts) == 1 and ts[0] == eprob.prob.tspan[1]           # :716
    out_u = sol.u
    if save_idxs is not None:                                          # :733-738
        idx = [save_idxs] if np.isscalar(save_idxs) else list(save_idxs)
        out_u = out_u[:, idx, :]
    out = EnsembleSolution(prob=eprob, alg=alg, t=ts, u=out_u, retcode=sol.retcode, engine=sol.engine, u0=u0m, p=p)
    no_start = (not save_start) and len(ts) > 0 and ts[0] == eprob.prob.tspan[0]   # :962
    eng = sol.engine

    def adjoint_sensitivity_backpass(Delta):
        if isinstance(Delta, AffineCost):
            dg = Delta
        else:
            D_ = Delta.u if isinstance(Delta, EnsembleSolution) else Delta
            if only_end and D_.ndim == 2:                                  # Delta may be a vector (:783-814)
                D_ = D_.reshape(1, *D_.shape)
            if save_idxs is not None:                                       # scatter into a full-d jump (:792-801)
                full = (np.zeros if not _is_torch(D_) else __import__("torch").zeros)((len(ts), d, eng.N), **({} if not _is_torch(D_) else {"dtype": D_.dtype, "device": D_.device}))
                full[:, idx, :] = D_
                D_ = full
            dg = D_
        # rrule path: Backsolve checkpoints = the saved times (forward saved only at saveat, :689-694)
        du0, dp = adjoint_sensitivities(sol, alg, sensealg=sensealg, t=ts, dgdu_discrete=dg, no_start=no_start,
                                        checkpoints=ts, row_dp=False, **{k: v for k, v in kwargs.items() if k in ("abstol", "reltol")})
        du0 = du0.reshape(u0_shape) if tuple(du0.shape) != u0_shape and int(np.prod(u0_shape)) == int(np.prod(du0.shape)) else du0
        dp = dp.reshape(tuple(p.shape))                                    # dp' -> size(tunables) (:980-986)
        if isinstance(originator, TrackerOriginator):
            return (NoTangent(), NoTangent(), du0, dp, NoTangent()) + tuple(NoTangent() for _ in args)
        return (NoTangent(), NoTangent(), NoTangent(), du0, dp, NoTangent()) + tuple(NoTangent() for _ in args)

    return out, adjoint_sensitivity_backpass
