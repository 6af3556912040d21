"""General-noise SDE families (examples/sde_noise_families.cuh) on the device, against the restatement of
tests/sde_noise_restatement.py, closed forms and the reference's own relations.

* The configuration matrix of sde_noise_restatement (the six example families x EM / EulerHeun x Backsolve with each
  checkpoint mode and Interpolating with and without no_start, EM + Backsolve excepted, x scalar affine, vector affine plus
  dgdp, explicit cost x shared and per-member p x regenerated, stored and caller-supplied noise x four save tables; every
  pair of levels and every reverse-kernel instantiation of every family): du0 and dp per member and component at 1e-12
  relative under the bound rules of test_gpu_sde_reference.py, in 40 digits for 3 members and in long double for all.
* The seam: sde_lv written in the general shape against the built-in sde_lv on identical inputs, at 1e-14.
* Convergence: Roessler and scalar-noise gradients, with caller-supplied increments from one fine path per member, reach
  the closed form at order about 1 as dt halves four times.
* The reference's relations on its configuration (T = 0.1, dt = 1e-4, u0 = [0.75, 0.5], p = [-1.5, 0.05, 0.2, 0.01], saves
  every 0.005, dg = u): InterpolatingAdjoint against BacksolveAdjoint and the Roessler gradient against its closed form.
* Two shards reproduce the unsharded run bitwise; an overflowing member gets status 1 and changes no other member.
* Refusals; the public API with noise_rate_prototype.

Observed on an H100 80GB HBM3 (700 W power limit): the matrix at most 0.40 of its bound (40 digits at most 2.3e-13); the seam
bitwise on EM + Interpolating, at most 9.3e-15 elsewhere; convergence orders 0.97-0.99; Interpolating ~ Backsolve on every
member but 14 % of the mixing family's dp (the ensemble as a whole within the reference's tolerance), the Roessler closed form
on 97 % of the members.  The module took 31 s there.
"""
import os
import sys

import numpy as np
import pytest

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(HERE)
for d in (ROOT, HERE):
    if d not in sys.path:
        sys.path.insert(0, d)

import sde_restatement as R
import sde_noise_restatement as Q

pytestmark = pytest.mark.gpu
TOL = 1e-12
N_MATRIX = 48


@pytest.fixture(scope="module")
def families():
    import scimlsensitivity_jl_b200 as b
    import __graft_entry__ as g
    for struct, name in g.SDE_NOISE_FAMILIES:
        so = os.path.join(ROOT, "examples", f"libb200fam_{name}.so")
        if not os.path.exists(so):
            so = b.build_family_plugin(os.path.join(ROOT, "examples", "sde_noise_families.cuh"), struct, name, out=so, sde=True, noise="general")
        b.register_family(so)
    return b


def _engine(b, c, inp, N, seed=0, traj_offset=0):
    u0, p, cost, dgdp, dLdu = inp
    sensealg, ckpt, no_start = R.SENSEALGS[c["sa"]]
    acost = None if cost[0] == "explicit" else b.AffineCost(cost[1], cost[2])
    kw = dict(no_start=no_start, checkpointing=ckpt != "never", ckpt_every_step=ckpt == "every")
    eng = b.DeviceEnsemble(c["family"], sensealg, c["stepper"], N, R.SAVEATS[c["saveat"]], (0.0, R.T_END), R.H,
                           shared_p=c["p"] == "shared", cost=acost, stored_noise=c["noise"] == "stored", seed=2000 + seed,
                           traj_offset=traj_offset, **kw)
    if dgdp is not None:
        eng.set_reverse(sensealg, cost=acost, dgdp=b.ParamAffine(dgdp[0], dgdp[1]), **kw)
    return eng


def _run(b, c, inp, seed=0, traj_offset=0):
    """-> (saved, dW, du0, dp) of one device run"""
    N = inp[0].shape[1]
    M = b.FAMILIES[c["family"]][2]
    eng = _engine(b, c, inp, N, seed, traj_offset)
    dW_in = np.sqrt(R.H) * np.random.default_rng(seed + 1).standard_normal((R.S_STEPS, M, N)) if c["noise"] == "dW" else None
    saved, status = eng.forward(inp[0], inp[1], dW=dW_in)
    assert (np.asarray(status) == 0).all()
    dW = np.array(eng.noise())
    assert dW.shape == (R.S_STEPS, M, N)
    if dW_in is not None:
        assert np.array_equal(dW, dW_in)
    du0, dp = [np.array(x) for x in eng.reverse(inp[4])]
    eng.close()
    return np.array(saved), dW, du0, dp


def _restated(kind, c, inp, dW, idx=None):
    u0, p, cost, dgdp, dLdu = inp
    sensealg, ckpt, no_start = R.SENSEALGS[c["sa"]]
    sel = (lambda a: a) if idx is None else (lambda a: a[..., idx])
    return Q.gradient(kind, c["family"], c["stepper"], sensealg, sel(u0), p if np.ndim(p) == 1 else sel(p), sel(dW), R.H,
                      R.SAVEATS[c["saveat"]], cost=cost, dLdu=None if dLdu is None else sel(dLdu), dgdp=dgdp, ckpt=ckpt,
                      no_start=no_start)


def _dgdp_part(c, inp):
    u0, p, cost, dgdp, dLdu = inp
    if dgdp is None:
        return None
    K = len(R.SAVEATS[c["saveat"]]) - (1 if c["sa"] == "interp_no_start" else 0)
    pm = np.asarray(p, dtype=np.float64)
    pm = np.repeat(pm[:, None], u0.shape[1], 1) if pm.ndim == 1 else pm
    return K * (np.asarray(dgdp[0])[:, None] * pm + np.asarray(dgdp[1])[:, None])


def _errors(c, du0, dp, ref_du0, ref_dp, idx=None, f64_shared=False, part=None):
    """as test_gpu_sde_reference._errors"""
    if f64_shared and c["p"] == "shared":
        dp = dp.sum(1)
    sel = (lambda a: a) if idx is None else (lambda a: a[..., idx])
    e = R.rel_err(sel(du0), ref_du0).max()
    if c["p"] == "shared":
        if idx is None:
            e = max(e, R.rel_err(dp, ref_dp.sum(1), None if part is None else part.sum(1)).max())
    else:
        e = max(e, R.rel_err(sel(dp), ref_dp, None if part is None else sel(part)).max())
    return e


@pytest.mark.parametrize("c", Q.config_matrix(), ids=R.label)
def test_device_matches_the_restatement(families, c):
    N = N_MATRIX
    inp = Q.problem(c, N, seed=3)
    saved, dW, du0, dp = _run(families, c, inp, seed=3, traj_offset=2 ** 32 - N // 2)
    idx = np.array([0, N // 2, N - 1])
    part = _dgdp_part(c, inp)
    mp_ = _restated("mp", c, inp, dW, idx)
    e_mp = _errors(c, du0, dp, mp_[0], mp_[1], idx, part=part)
    ld = _restated("ld", c, inp, dW)
    assert R.rel_err(ld[0][:, idx], mp_[0]).max() < 1e-15
    f64 = _restated("f64", c, inp, dW)
    tol = max(TOL, 4 * _errors(c, f64[0], f64[1], ld[0], ld[1], f64_shared=True, part=part))
    e_ld = _errors(c, du0, dp, ld[0], ld[1], part=part)
    us = ld[2][np.rint(R.SAVEATS[c["saveat"]] / R.H).astype(int)]
    e_u = np.abs(saved - us).max() / np.abs(us).max()
    print(f"{R.label(c)}: 40 digits {e_mp:.2e}, long double {e_ld:.2e}, bound {tol:.2e}, saved {e_u:.2e}")
    assert e_mp < tol and e_ld < tol and e_u < 1e-13


@pytest.mark.parametrize("stepper,sa", [("em", "interp"), ("euler_heun", "bs_save"), ("euler_heun", "bs_every"), ("euler_heun", "interp_no_start")])
def test_general_form_of_lv_agrees_with_the_builtin(families, stepper, sa):
    c = dict(family="sde_lv", stepper=stepper, sa=sa, cost="vector_dgdp", p="member", noise="regen", saveat="full")
    inp = R.problem(c, 64, seed=7)
    ref = _run(families, c, inp, seed=7)
    got = _run(families, dict(c, family="sde_lv_general"), inp, seed=7)
    assert np.array_equal(ref[1], got[1])                                      # the same Philox increments
    e = [R.rel_err(g.reshape(-1, 64), r.reshape(-1, 64)).max() for g, r in zip((got[0], got[2], got[3]), (ref[0], ref[2], ref[3]))]
    print(f"{stepper} {sa}: saved {e[0]:.2e}, du0 {e[1]:.2e}, dp {e[2]:.2e}")
    assert max(e) <= 1e-14


@pytest.mark.parametrize("family", ["sde_roessler", "sde_scalar"])
def test_device_gradients_converge_to_the_closed_form(families, family):
    b = families
    _, _, D, P, M = Q.FAMILIES[family]
    N, T, SF = 256, 0.5, 1024
    ts = np.array([0.125, 0.25, 0.375, 0.5])
    u0 = np.asarray(Q.U0_NOMINAL[family])[:, None] * np.ones((D, N))
    p = np.asarray(Q.P_NOMINAL[family])
    dWf = np.sqrt(T / SF) * np.random.default_rng(15).standard_normal((SF, M, N))
    Wf = np.concatenate([np.zeros((1, M, N)), np.cumsum(dWf, 0)])
    at = (ts / T * SF).round().astype(int)
    ref = [Q.closed_gradient(family, u0[:, i], p, Wf[at][:, :, i], ts) for i in range(N)]
    ref_du0, ref_dp = np.array([r[0] for r in ref]).T, np.array([r[1] for r in ref]).T
    for sa in ("backsolve", "interpolating"):
        errs = []
        for S in (32, 64, 128, 256, 512):
            eng = b.DeviceEnsemble(family, sa, "euler_heun", N, ts, (0.0, T), T / S, shared_p=False, cost=b.AffineCost(1.0, 0.0))
            eng.forward(u0, np.repeat(p[:, None], N, 1), dW=dWf.reshape(S, SF // S, M, N).sum(1))
            du0, dp = [np.array(x) for x in eng.reverse()]
            eng.close()
            e = lambda x, r: (np.abs(x - r).max(0) / np.abs(r).max(0)).mean()
            errs.append(e(du0, ref_du0) + e(dp, ref_dp))
        order = -np.polyfit(np.arange(len(errs)), np.log2(errs), 1)[0]
        print(f"{family} {sa}: errors {np.array(errs)}, order {order:.2f}")
        assert 0.8 < order < 1.3


def _julia_isapprox(a, b_, rtol):
    return np.linalg.norm(a - b_) <= rtol * max(np.linalg.norm(a), np.linalg.norm(b_))


def test_reference_relations_on_the_reference_configuration(families):
    """test/SDE2/sde_nondiag_stratonovich.jl:139-166, 286-287, 399-473.  The reference checks one path; here every member is
    one path, and the relation must hold on the ensemble as a whole and on 80 % of its members (with this seed, in the
    restatement: Interpolating ~ Backsolve on all members but 14 % of the mixing family's dp, the closed form on 97 %)."""
    b = families
    N, T, dt = 64, 0.1, 1e-4
    ts = np.linspace(0.0, T, 21)
    u0 = np.repeat(np.array([[0.75], [0.5]]), N, 1)
    p = np.array([-1.5, 0.05, 0.2, 0.01])
    res = {}
    for fam in ("sde_roessler", "sde_mixing"):
        for sa in ("backsolve", "interpolating"):
            eng = b.DeviceEnsemble(fam, sa, "euler_heun", N, ts, (0.0, T), dt, shared_p=False, cost=b.AffineCost(1.0, 0.0), seed=100)
            eng.forward(u0, np.repeat(p[:, None], N, 1))
            du0, dp = [np.array(x) for x in eng.reverse()]
            res[fam, sa] = (du0, dp, np.array(eng.noise()))
            eng.close()
    for fam, (ru, rp) in (("sde_roessler", (1e-5, 1e-4)), ("sde_mixing", (1e-5, 1e-5))):
        (bu, bp, _), (iu, ip, _) = res[fam, "backsolve"], res[fam, "interpolating"]
        ok_u = np.mean([_julia_isapprox(iu[:, i], bu[:, i], ru) for i in range(N)])
        ok_p = np.mean([_julia_isapprox(ip[:, i], bp[:, i], rp) for i in range(N)])
        print(f"{fam}: Interpolating ~ Backsolve on {ok_u:.0%} (du0) and {ok_p:.0%} (dp) of the members")
        assert ok_u >= 0.8 and ok_p >= 0.8 and _julia_isapprox(iu, bu, ru) and _julia_isapprox(ip, bp, rp)
    W = np.concatenate([np.zeros((1, 2, N)), np.cumsum(res["sde_roessler", "backsolve"][2], 0)])[np.rint(ts / dt).astype(int)]
    bu, bp, _ = res["sde_roessler", "backsolve"]
    ok = np.mean([all(_julia_isapprox(x, y, 1e-4) for x, y in zip((bu[:, i], bp[:, i]), Q.closed_gradient("sde_roessler", u0[:, i], p, W[:, :, i], ts)))
                  for i in range(N)])
    print(f"Roessler gradient within 1e-4 of the closed form on {ok:.0%} of the members")
    assert ok >= 0.8


@pytest.mark.parametrize("family", ["sde_nonsquare", "sde_scalar"])
def test_two_shards_reproduce_the_unsharded_run(families, family):
    c = dict(family=family, stepper="euler_heun", sa="bs_save", cost="vector_dgdp", p="member", noise="regen", saveat="no_T")
    N = 64
    inp = Q.problem(c, N, seed=30)
    whole = _run(families, c, inp, seed=30)
    cut = lambda a, s: None if a is None else (a[..., s] if np.ndim(a) > 1 else a)
    for lo in (0, N // 2):
        s = slice(lo, lo + N // 2)
        half = _run(families, c, tuple(cut(x, s) if k in (0, 1, 4) else x for k, x in enumerate(inp)), seed=30, traj_offset=lo)
        for x, y, what in zip(whole, half, ("saved", "get_noise", "du0", "dp")):
            assert np.array_equal(x[..., s], y), what


def test_an_overflowing_member_gets_status_1_and_changes_no_other(families):
    b = families
    c = dict(family="sde_scalar", stepper="euler_heun", sa="interp", cost="scalar", p="member", noise="regen", saveat="full")
    u0, p, _, _, _ = Q.problem(c, 8, seed=50)
    out = []
    for bad in (False, True):
        uu = u0.copy()
        if bad:
            uu[:, 3] = 1e308
        eng = b.DeviceEnsemble("sde_scalar", "interpolating", "euler_heun", 8, R.SAVEATS["full"], (0.0, R.T_END), R.H, shared_p=False,
                               cost=b.AffineCost(1.0, 0.0))
        saved, status = eng.forward(uu, p)
        out.append((np.asarray(status).copy(), np.array(saved)) + tuple(np.array(x) for x in eng.reverse()))
        eng.close()
    assert list(out[0][0]) == [0] * 8 and list(out[1][0]) == [0, 0, 0, 1, 0, 0, 0, 0]
    assert not np.isfinite(out[1][2][:, 3]).all() and not np.isfinite(out[1][3][:, 3]).all()
    keep = np.arange(8) != 3
    for a, b_ in zip(out[0][1:], out[1][1:]):
        assert np.array_equal(a[..., keep], b_[..., keep])


def test_steppers_and_sensealgs_a_general_family_refuses(families):
    b = families
    t = R.SAVEATS["full"]
    for stepper, dt in (("tsit5_fixed", R.H), ("rosenbrock23", 0.0)):
        with pytest.raises(b.B200AdjError) as e:
            b.DeviceEnsemble("sde_roessler", "interpolating", stepper, 8, t, (0.0, R.T_END), dt)
        assert e.value.code == -1, (stepper, e.value)
    for sa in ("gauss", "quadrature", "gauss_kronrod"):
        with pytest.raises(b.B200AdjError) as e:
            b.DeviceEnsemble("sde_mixing", sa, "euler_heun", 8, t, (0.0, R.T_END), R.H)
        assert e.value.code == -2, (sa, e.value)
    with pytest.raises(b.B200AdjError) as e:                                   # the C ABI refuses it too, not only the host
        b.DeviceEnsemble("sde_nonsquare", "backsolve", "em", 8, t, (0.0, R.T_END), R.H)
    assert e.value.code == -2 and "EM + BacksolveAdjoint" in str(e.value)
    eng = b.DeviceEnsemble("sde_nonsquare", "interpolating", "em", 8, t, (0.0, R.T_END), R.H)
    with pytest.raises(b.B200AdjError) as e:
        eng.set_reverse("backsolve")
    assert e.value.code == -2
    eng.close()


def test_public_api_with_noise_rate_prototype(families):
    b = families
    fam, D, P, M, N = "sde_nonsquare", 3, 2, 2, 24
    ts = R.SAVEATS["no_T"]
    rng = np.random.default_rng(40)
    u0s = np.asarray(Q.U0_NOMINAL[fam])[:, None] * np.exp(0.05 * rng.standard_normal((D, N)))
    ps = np.asarray(Q.P_NOMINAL[fam])[:, None] * np.exp(0.02 * rng.standard_normal((P, N)))
    prob = b.SDEProblem(fam, u0s[:, 0], (0.0, R.T_END), ps[:, 0], seed=77, noise_rate_prototype=np.zeros((D, M)))
    eprob = b.EnsembleProblem(prob, prob_func=lambda pr, i: (u0s[:, i], ps[:, i]))
    alg = b.EulerHeun(dt=R.H)
    sol = b.solve(eprob, alg, b.EnsembleB200(device=0), trajectories=N, saveat=ts, sensealg=b.B200Adjoint(b.BacksolveAdjoint(noisemixing=True)))
    assert (np.asarray(sol.retcode) == 0).all()
    dW = np.array(sol.engine.noise())
    du0, dp = b.adjoint_sensitivities(sol, alg, t=ts, dgdu_discrete=b.AffineCost(1.0, -0.25), sensealg=b.BacksolveAdjoint(noisemixing=True))
    args = (fam, "euler_heun", "backsolve", u0s, ps, dW, R.H, ts)
    ld, f64 = [Q.gradient(k, *args, cost=("affine", 1.0, -0.25), ckpt="every") for k in ("ld", "f64")]
    us = ld[2][np.rint(ts / R.H).astype(int)]
    assert R.rel_err(np.asarray(sol.u).reshape(-1, N), us.reshape(-1, N)).max() < 1e-13
    tol = max(TOL, 4 * max(R.rel_err(f64[0], ld[0]).max(), R.rel_err(f64[1], ld[1]).max()))
    assert max(R.rel_err(du0, ld[0]).max(), R.rel_err(dp, ld[1]).max()) < tol
    with pytest.raises(NotImplementedError, match="EM \\+ BacksolveAdjoint"):
        b.adjoint_sensitivities(b.solve(eprob, b.EM(dt=R.H), b.EnsembleB200(device=0), trajectories=N, saveat=ts), b.EM(dt=R.H), t=ts,
                                dgdu_discrete=b.AffineCost(1.0, 0.0), sensealg=b.BacksolveAdjoint())
    # the rrule: EM + InterpolatingAdjoint, cotangent Delta[K][D][N] at the save times
    out, pullback = b._concrete_solve_adjoint(prob, b.EM(dt=R.H), b.B200Adjoint(b.InterpolatingAdjoint()), u0s, ps, saveat=ts)
    Delta = rng.uniform(0.5, 1.5, (len(ts), D, N))
    tang = pullback(Delta)
    du0r, dpr = np.asarray(tang[3]), np.asarray(tang[4])
    dW2 = np.array(out.engine.noise())
    assert np.array_equal(dW2, dW)
    args = (fam, "em", "interpolating", u0s, ps, dW2, R.H, ts)
    ld, f64 = [Q.gradient(k, *args, cost=("explicit",), dLdu=Delta) for k in ("ld", "f64")]
    tol = max(TOL, 4 * max(R.rel_err(f64[0], ld[0]).max(), R.rel_err(f64[1], ld[1]).max()))
    assert du0r.shape == (D, N) and dpr.shape == (P, N)
    assert max(R.rel_err(du0r, ld[0]).max(), R.rel_err(dpr, ld[1]).max()) < tol
