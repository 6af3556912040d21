"""User diagonal-noise SDE families as plug-ins (csrc/family_plugin.inc with B200ADJ_FAMILY_SDE) on EM / EulerHeun with
BacksolveAdjoint / InterpolatingAdjoint.

* The seam is bit for bit: SdeLotkaVolterra and SdeLinear2 built as plug-ins straight from the library's csrc/families.cuh
  reproduce the built-in sde_lv / sde_linear exactly (saved states, get_noise, du0, dp) over the configuration matrix of
  tests/sde_restatement.py (EM / EulerHeun x Backsolve with checkpoints at the save times, every step or never, and
  Interpolating with and without no_start x scalar affine, vector affine plus dgdp, explicit cost x shared and per-member p x
  regenerated, stored and caller-supplied noise x four save grids; every pair of levels).
* The example families of examples/sde_families.cuh (SdeFoodChain3: d = 3, P = 6, saturating noise with g'' != 0 and one
  half-used Philox pair; SdeOscillator4: d = 4, P = 8, the registry's limits) against the restatement, which takes every
  derivative of the Python f and g below -- the Ito correction included -- from complex steps and dual numbers: du0 and dp per
  member and component at 1e-12 relative with the bound rules of tests/test_gpu_sde_reference.py, in 40 digits for 3 members
  and in long double for all, over the same configuration factors.
* The ITO instantiation that runs: Backsolve + EM lies >= 100 bounds from the restatement with the half Ito correction;
  Backsolve + EulerHeun and Interpolating (EM and EulerHeun) match the untransformed drift and lie >= 100 bounds from the
  transformed one.
* The public API (SDEProblem through EnsembleProblem(prob_func), solve, adjoint_sensitivities and _concrete_solve_adjoint)
  and sharding: two shards at traj_offset 0 and N/2 reproduce the unsharded states, increments and gradients bitwise.
* Refusals: an SDE plug-in on Tsit5 / Rosenbrock23 and an ODE plug-in on EM are INVALID, Gauss / Quadrature / GaussKronrod
  on an SDE plug-in UNSUPPORTED; an overflowing member gets status 1 as with the built-ins.  (b200adj_family_noise, the
  stale-plug-in refusal and the host's noisemixing refusal need no GPU: tests/test_sde_family_plugin_build.py.)
"""
import os
import sys
from concurrent.futures import ThreadPoolExecutor

import numpy as np
import pytest

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(HERE)
for d in (ROOT, HERE):
    if d not in sys.path:
        sys.path.insert(0, d)

import sde_restatement as R

import scimlsensitivity_jl_b200 as b
from scimlsensitivity_jl_b200 import _lib

pytestmark = pytest.mark.gpu
TOL = 1e-12
EXAMPLES = os.path.join(ROOT, "examples")


# ---- the example families restated in Python (examples/sde_families.cuh); derivatives come from R's complex steps ----

def _recip(x):
    """1 / x, for the dual numbers of R.ito_drift as well"""
    return R.Dual(1 / x.a, -x.b / (x.a * x.a)) if isinstance(x, R.Dual) else 1 / x


def f_chain3(u, p):
    return [u[0] * (p[0] - u[1]), u[1] * (u[0] - p[1] - u[2]), u[2] * (u[1] - p[2])]


def g_chain3(u, p):
    return [p[3 + i] * u[i] * _recip(1 + u[i] * u[i]) for i in range(3)]


def f_osc4(u, p):
    return [u[1], -p[0] * u[0] - p[1] * u[1] + p[2] * (u[2] - u[0]), u[3], -p[3] * u[2] * u[2] * u[2] + p[2] * (u[0] - u[2])]


def g_osc4(u, p):
    return [p[4 + i] * (1 + u[i] * u[i]) for i in range(4)]


R.FAMILIES["sde_chain3"] = (f_chain3, g_chain3, 3, 6)
R.FAMILIES["sde_osc4"] = (f_osc4, g_osc4, 4, 8)
# the Ito-transformed drift as a family's own drift: what EulerHeun / Interpolating would compute on the ITO = true instantiation
R.FAMILIES["sde_chain3_ito"] = (R.ito_drift(f_chain3, g_chain3, 3), g_chain3, 3, 6)

NOMINAL = {"sde_lv": (R.U0_NOMINAL["sde_lv"], R.P_NOMINAL["sde_lv"]), "sde_linear": (R.U0_NOMINAL["sde_linear"], R.P_NOMINAL["sde_linear"]),
           "sde_chain3": ([1.0, 0.5, 0.8], [1.2, 0.8, 0.6, 0.3, 0.25, 0.35]),
           "sde_osc4": ([0.8, 0.1, -0.5, 0.3], [1.5, 0.3, 0.4, 1.0, 0.08, 0.1, 0.06, 0.12])}
SEAM = {"sde_lv": ("SdeLotkaVolterra", "sde_lv_seam"), "sde_linear": ("SdeLinear2", "sde_linear_seam")}
NEW = {"sde_lv": "sde_chain3", "sde_linear": "sde_osc4"}      # the matrix's family factor, mapped onto the example families


def _register(so, build):
    """register a prebuilt plug-in; one built against other headers is rebuilt (into a temporary directory)"""
    if os.path.exists(so):
        try:
            return b.register_family(so)
        except b.B200AdjError:
            pass
    return b.register_family(build())


@pytest.fixture(scope="module")
def families(tmp_path_factory):
    tmp = str(tmp_path_factory.mktemp("sde_plugins"))
    fams = (("SdeFoodChain3", "sde_chain3"), ("SdeOscillator4", "sde_osc4"))
    for struct, name in fams:
        _register(os.path.join(EXAMPLES, f"libb200fam_{name}.so"),
                  lambda: b.build_family_plugin(os.path.join(EXAMPLES, "sde_families.cuh"), struct, name,
                                                out=os.path.join(tmp, f"libb200fam_{name}.so"), sde=True))
    _register(os.path.join(EXAMPLES, "libb200fam_vanderpol.so"),
              lambda: b.build_family_plugin(os.path.join(EXAMPLES, "vanderpol_family.cuh"), "VanDerPol", "vanderpol",
                                            out=os.path.join(tmp, "libb200fam_vanderpol.so")))
    # the built-in SDE families, compiled as plug-ins from the library's own header (no copy)
    with ThreadPoolExecutor(max_workers=2) as pool:
        sos = list(pool.map(lambda s: b.build_family_plugin(os.path.join(_lib._CSRC, "families.cuh"), s[0], s[1],
                                                            out=os.path.join(tmp, f"libb200fam_{s[1]}.so"), sde=True), SEAM.values()))
    for so in sos:
        b.register_family(so)
    assert b.FAMILIES["sde_chain3"] == (3, 6, 3) and b.FAMILIES["sde_osc4"] == (4, 8, 4)
    assert b.FAMILIES["sde_lv_seam"] == b.FAMILIES["sde_lv"] and b.FAMILIES["sde_linear_seam"] == b.FAMILIES["sde_linear"]
    return True


# ---- one device run and its restatement ----------------------------------------------------------------------------

def _problem(c, N, seed):
    """u0[D][N], p ([P] or [P][N]), cost tuple, dgdp or None, dLdu or None of a configuration"""
    rng = np.random.default_rng(seed)
    fam = c["family"]
    _, _, D, P = R.FAMILIES[fam]
    u0n, pn = NOMINAL[fam]
    u0 = np.asarray(u0n, dtype=np.float64)[:, None] * np.exp(0.05 * rng.standard_normal((D, N)))
    p = np.asarray(pn, dtype=np.float64)
    if c["p"] == "member":
        p = p[:, None] * np.exp(0.02 * rng.standard_normal((P, N)))
    K = len(R.SAVEATS[c["saveat"]])
    dLdu = rng.uniform(0.5, 1.5, (K, D, N)) if c["cost"] == "explicit" else None
    cost = {"explicit": ("explicit",), "scalar": ("affine", 1.0, -0.25),
            "vector_dgdp": ("affine", np.linspace(1.0, 0.5, D), np.linspace(-0.3, 0.2, D))}[c["cost"]]
    dgdp = (np.linspace(0.2, 0.7, P), np.linspace(-0.1, 0.15, P)) if c["cost"] == "vector_dgdp" else None
    return u0, p, cost, dgdp, dLdu


def _members(inp, sl):
    """the inputs of members sl"""
    u0, p, cost, dgdp, dLdu = inp
    return u0[:, sl], (p if np.ndim(p) == 1 else p[:, sl]), cost, dgdp, (None if dLdu is None else dLdu[..., sl])


def _run(c, inp, family=None, seed=0, traj_offset=0, dW_in=None):
    """-> (saved, dW, du0, dp) of one device run of configuration c on `family` (default: c's)"""
    u0, p, cost, dgdp, dLdu = inp
    N = u0.shape[1]
    sensealg, ckpt, no_start = R.SENSEALGS[c["sa"]]
    acost = None if cost[0] == "explicit" else b.AffineCost(cost[1], cost[2])
    kw = dict(no_start=no_start, checkpointing=ckpt != "never", ckpt_every_step=ckpt == "every")
    eng = b.DeviceEnsemble(family or c["family"], sensealg, c["stepper"], N, R.SAVEATS[c["saveat"]], (0.0, R.T_END), R.H,
                           shared_p=c["p"] == "shared", cost=acost, stored_noise=c["noise"] == "stored", seed=1000 + seed,
                           traj_offset=traj_offset, **kw)
    if dgdp is not None:
        eng.set_reverse(sensealg, cost=acost, dgdp=b.ParamAffine(dgdp[0], dgdp[1]), **kw)
    saved, status = eng.forward(u0, p, dW=dW_in)
    assert (np.asarray(status) == 0).all()
    dW = np.array(eng.noise())
    if dW_in is not None:
        assert np.array_equal(dW, dW_in)
    du0, dp = [np.array(x) for x in eng.reverse(dLdu)]
    eng.close()
    return np.array(saved), dW, du0, dp


def _dw_in(c, N, D, seed):
    return np.sqrt(R.H) * np.random.default_rng(seed + 1).standard_normal((R.S_STEPS, D, N)) if c["noise"] == "dW" else None


def _restated(kind, c, inp, dW, idx=None, family=None, variant=None):
    u0, p, cost, dgdp, dLdu = inp
    sensealg, ckpt, no_start = R.SENSEALGS[c["sa"]]
    sel = (lambda a: a) if idx is None else (lambda a: a[..., idx])
    return R.gradient(kind, family or c["family"], c["stepper"], sensealg, sel(u0), p if np.ndim(p) == 1 else sel(p), sel(dW), R.H,
                      R.SAVEATS[c["saveat"]], cost=cost, dLdu=None if dLdu is None else sel(dLdu), dgdp=dgdp, ckpt=ckpt,
                      no_start=no_start, variant=variant)[:2]


def _dgdp_part(c, inp):
    """the parameter part njump (c p + e) of dp per member (None without dgdp)"""
    u0, p, cost, dgdp, dLdu = inp
    if dgdp is None:
        return None
    K = len(R.SAVEATS[c["saveat"]]) - (1 if c["sa"] == "interp_no_start" else 0)
    pm = np.asarray(p, dtype=np.float64)
    pm = np.repeat(pm[:, None], u0.shape[1], 1) if pm.ndim == 1 else pm
    return K * (np.asarray(dgdp[0])[:, None] * pm + np.asarray(dgdp[1])[:, None])


def _errors(c, du0, dp, ref_du0, ref_dp, idx=None, f64_shared=False, part=None):
    """largest floored relative error of du0 and dp (dp summed over the members under shared p)"""
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


def _bound(c, inp, dW, ld):
    """1e-12, or 4x the float64 restatement's own distance from the long-double one where that is larger"""
    f64 = _restated("f64", c, inp, dW)
    return max(TOL, 4 * _errors(c, f64[0], f64[1], ld[0], ld[1], f64_shared=True, part=_dgdp_part(c, inp)))


# ---- 1. the seam ---------------------------------------------------------------------------------------------------

@pytest.mark.parametrize("c", R.config_matrix(), ids=R.label)
def test_plugin_from_families_cuh_is_the_builtin_family_bitwise(families, c):
    N = 40
    inp = _problem(c, N, seed=21)
    dW_in = _dw_in(c, N, R.FAMILIES[c["family"]][2], 21)
    a = _run(c, inp, seed=21, traj_offset=2 ** 32 - N // 2, dW_in=dW_in)
    p = _run(c, inp, family=SEAM[c["family"]][1], seed=21, traj_offset=2 ** 32 - N // 2, dW_in=dW_in)
    for x, y, what in zip(a, p, ("saved", "get_noise", "du0", "dp")):
        assert np.array_equal(x, y), what


# ---- 2. the example families against the restatement ----------------------------------------------------------------

NEW_MATRIX = [dict(c, family=NEW[c["family"]]) for c in R.config_matrix()]
N_MATRIX = 48


@pytest.mark.parametrize("c", NEW_MATRIX, ids=R.label)
def test_example_family_matches_the_restatement(families, c):
    N = N_MATRIX
    D = R.FAMILIES[c["family"]][2]
    inp = _problem(c, N, seed=3)
    _, dW, du0, dp = _run(c, inp, seed=3, traj_offset=2 ** 32 - N // 2, dW_in=_dw_in(c, N, D, 3))
    idx = np.array([0, N // 2, N - 1])
    part = _dgdp_part(c, inp)
    mp_ = _restated("mp", c, inp, dW, idx)
    e_mp = _errors(c, du0, dp, mp_[0], mp_[1], idx, part=part)
    ld = _restated("ld", c, inp, dW)
    assert R.rel_err(ld[0][:, idx], mp_[0]).max() < 1e-15          # long double stands in for 40 digits
    tol = _bound(c, inp, dW, ld)
    e_ld = _errors(c, du0, dp, ld[0], ld[1], part=part)
    print(f"{R.label(c)}: 40 digits {e_mp:.2e}, long double {e_ld:.2e}, bound {tol:.2e}")
    assert e_mp < tol and e_ld < tol


# ---- 3. the ITO instantiation that runs --------------------------------------------------------------------------

@pytest.mark.parametrize("stepper,sa", [("em", "bs_save"), ("euler_heun", "bs_save"), ("em", "interp"), ("euler_heun", "interp")])
def test_the_ito_instantiation_is_the_one_that_runs(families, stepper, sa):
    c = dict(family="sde_chain3", stepper=stepper, sa=sa, cost="scalar", p="member", noise="regen", saveat="full")
    inp = _problem(c, 64, seed=4)
    _, dW, du0, dp = _run(c, inp, seed=4)
    ok = _restated("ld", c, inp, dW)
    tol = _bound(c, inp, dW, ok)
    assert _errors(c, du0, dp, ok[0], ok[1]) < tol
    if stepper == "em" and sa == "bs_save":
        bad = _restated("ld", c, inp, dW, variant="half_ito")          # the 1/2-factor Ito correction
    else:
        bad = _restated("ld", c, inp, dW, family="sde_chain3_ito")      # the transformed drift where the plain one belongs
    sep = _errors(c, du0, dp, bad[0], bad[1]) / tol
    print(f"{stepper} {sa}: the device lies {sep:.3g} bounds from the wrong drift")
    assert sep >= 100


# ---- 4. public API and sharding ------------------------------------------------------------------------------------

def test_public_api_solve_adjoint_sensitivities_and_rrule(families):
    fam, D, P, N = "sde_osc4", 4, 8, 24
    ts = R.SAVEATS["no_T"]
    rng = np.random.default_rng(40)
    u0n, pn = NOMINAL[fam]
    u0s = np.asarray(u0n)[:, None] * np.exp(0.05 * rng.standard_normal((D, N)))
    ps = np.asarray(pn)[:, None] * np.exp(0.02 * rng.standard_normal((P, N)))
    prob = b.SDEProblem(fam, u0s[:, 0], (0.0, R.T_END), ps[:, 0], seed=77)
    eprob = b.EnsembleProblem(prob, prob_func=lambda pr, i: (u0s[:, i], ps[:, i]))
    alg = b.EM(dt=R.H)
    sol = b.solve(eprob, alg, b.EnsembleB200(device=0), trajectories=N, saveat=ts, sensealg=b.B200Adjoint(b.BacksolveAdjoint()))
    assert (np.asarray(sol.retcode) == 0).all()
    dW = np.array(sol.engine.noise())
    du0, dp = b.adjoint_sensitivities(sol, alg, t=ts, dgdu_discrete=b.AffineCost(1.0, -0.25), sensealg=b.BacksolveAdjoint())
    args = (fam, "em", "backsolve", u0s, ps, dW, R.H, ts)
    ld, f64 = [R.gradient(k, *args, cost=("affine", 1.0, -0.25), ckpt="every") for k in ("ld", "f64")]
    us = ld[2][np.rint(ts / R.H).astype(int)]
    assert R.rel_err(np.asarray(sol.u).reshape(-1, N), us.reshape(-1, N)).max() < 1e-13
    tol = max(TOL, 4 * max(R.rel_err(f64[0], ld[0]).max(), R.rel_err(f64[1], ld[1]).max()))
    assert max(R.rel_err(du0, ld[0]).max(), R.rel_err(dp, ld[1]).max()) < tol
    # the rrule: EulerHeun + InterpolatingAdjoint, cotangent Delta[K][D][N] at the save times
    out, pullback = b._concrete_solve_adjoint(prob, b.EulerHeun(dt=R.H), b.B200Adjoint(b.InterpolatingAdjoint()), u0s, ps, saveat=ts)
    Delta = rng.uniform(0.5, 1.5, (len(ts), D, N))
    tang = pullback(Delta)
    du0r, dpr = np.asarray(tang[3]), np.asarray(tang[4])
    dW2 = np.array(out.engine.noise())
    assert np.array_equal(dW2, dW)                                       # same seed, same members: the same increments
    args = (fam, "euler_heun", "interpolating", u0s, ps, dW2, R.H, ts)
    ld, f64 = [R.gradient(k, *args, cost=("explicit",), dLdu=Delta) for k in ("ld", "f64")]
    tol = max(TOL, 4 * max(R.rel_err(f64[0], ld[0]).max(), R.rel_err(f64[1], ld[1]).max()))
    assert du0r.shape == (D, N) and dpr.shape == (P, N)
    assert max(R.rel_err(du0r, ld[0]).max(), R.rel_err(dpr, ld[1]).max()) < tol


@pytest.mark.parametrize("family", ["sde_chain3", "sde_osc4"])
def test_two_shards_reproduce_the_unsharded_run(families, family):
    c = dict(family=family, stepper="euler_heun", sa="bs_save", cost="vector_dgdp", p="member", noise="regen", saveat="no_T")
    N = 64
    inp = _problem(c, N, seed=30)
    whole = _run(c, inp, seed=30)
    halves = [_run(c, _members(inp, slice(lo, lo + N // 2)), seed=30, traj_offset=lo) for lo in (0, N // 2)]
    for x, y0, y1, what in zip(whole, *halves, ("saved", "get_noise", "du0", "dp")):
        assert np.array_equal(x, np.concatenate([y0, y1], axis=-1)), what


# ---- 5. refusals and status --------------------------------------------------------------------------------------

def test_steppers_and_sensealgs_an_sde_plugin_refuses(families):
    t = R.SAVEATS["full"]
    for stepper, dt in (("tsit5_fixed", R.H), ("rosenbrock23", 0.0)):
        with pytest.raises(b.B200AdjError) as e:
            b.DeviceEnsemble("sde_chain3", "interpolating", stepper, 8, t, (0.0, R.T_END), dt)
        assert e.value.code == -1, (stepper, e.value)
    with pytest.raises(b.B200AdjError) as e:
        b.DeviceEnsemble("vanderpol", "backsolve", "em", 8, t, (0.0, R.T_END), R.H)
    assert e.value.code == -1
    for sa in ("gauss", "quadrature", "gauss_kronrod"):
        with pytest.raises(b.B200AdjError) as e:
            b.DeviceEnsemble("sde_osc4", sa, "em", 8, t, (0.0, R.T_END), R.H)
        assert e.value.code == -2, (sa, e.value)


@pytest.mark.parametrize("family", ["sde_lv", "sde_chain3", "sde_osc4"])
def test_an_overflowing_member_gets_status_1(families, family):
    c = dict(family=family, stepper="em", sa="bs_save", cost="scalar", p="shared", noise="regen", saveat="full")
    u0, p, _, _, _ = _problem(c, 8, seed=50)
    u0[:, 3] = 1e200
    eng = b.DeviceEnsemble(family, "backsolve", "em", 8, R.SAVEATS["full"], (0.0, R.T_END), R.H, cost=b.AffineCost(1.0, 0.0))
    _, status = eng.forward(u0, p)
    eng.close()
    assert list(np.asarray(status)) == [0, 0, 0, 1, 0, 0, 0, 0]
