"""Self-checks of the general-noise restatement (tests/sde_noise_restatement.py), without a GPU.

* Written in the general shape (a 2 x 2 diagonal G), sde_lv and sde_linear reproduce sde_restatement.reverse to 1e-15 over
  its whole configuration matrix, EM + BacksolveAdjoint included: the transformed drift f - J_{vec G}' vec G is the Ito
  correction for diagonal noise that does not mix.
* On one fine Brownian path per member (the coarse increments are sums of fine ones), the EulerHeun gradients of both
  sensealgs converge at order about 1 as dt halves four times, to closed forms of the Stratonovich solutions: the scalar
  linear SDE analytically, Roessler's non-diagonal example through scipy.linalg.expm_frechet, the non-square one per
  component.
* The mixing family has no closed form: its adjoint gradient approaches central differences of the restated forward solve
  at O(dt).
* Long double agrees with 40 digits on every example family.
"""
import os
import sys

import numpy as np
import pytest

HERE = os.path.dirname(os.path.abspath(__file__))
if HERE not in sys.path:
    sys.path.insert(0, HERE)

import sde_restatement as R
import sde_noise_restatement as Q

T_CONV, S_FINE = 0.5, 1024
S_COARSE = (32, 64, 128, 256, 512)
TS_CONV = np.array([0.125, 0.25, 0.375, 0.5])


@pytest.mark.parametrize("c", R.config_matrix(), ids=R.label)
def test_general_form_reproduces_the_diagonal_restatement(c):
    N = 4
    u0, p, cost, dgdp, dLdu = R.problem(c, N, seed=21)
    sensealg, ckpt, no_start = R.SENSEALGS[c["sa"]]
    dW = np.sqrt(R.H) * np.random.default_rng(22).standard_normal((R.S_STEPS, 2, N))
    args = dict(cost=cost, dLdu=dLdu, dgdp=dgdp, ckpt=ckpt, no_start=no_start)
    ref = R.gradient("ld", c["family"], c["stepper"], sensealg, u0, p, dW, R.H, R.SAVEATS[c["saveat"]], **args)
    got = Q.gradient("ld", Q.TWIN[c["family"]], c["stepper"], sensealg, u0, p, dW, R.H, R.SAVEATS[c["saveat"]], **args)
    assert np.abs(got[2] - ref[2]).max() <= 1e-15 * np.abs(ref[2]).max()
    assert R.rel_err(got[0], ref[0]).max() < 1e-15
    assert R.rel_err(got[1], ref[1]).max() < 1e-15


def _fine_path(M, N, seed):
    dWf = np.sqrt(T_CONV / S_FINE) * np.random.default_rng(seed).standard_normal((S_FINE, M, N))
    return dWf, np.concatenate([np.zeros((1, M, N)), np.cumsum(dWf, 0)])


def _order(errs):
    """least-squares slope of log2 error against log2 dt"""
    return -np.polyfit(np.arange(len(errs)), np.log2(errs), 1)[0]


def _err(du0, dp, ref_du0, ref_dp):
    """mean over members of the largest component error of du0 and of dp, relative to the member's largest component"""
    e = lambda x, r: (np.abs(x - r).max(0) / np.abs(r).max(0)).mean()
    return e(du0, ref_du0) + e(dp, ref_dp)


@pytest.mark.parametrize("sensealg", ["backsolve", "interpolating"])
@pytest.mark.parametrize("family", ["sde_scalar", "sde_roessler", "sde_nonsquare"])
def test_eulerheun_gradients_converge_to_the_closed_form(family, sensealg):
    _, _, D, P, M = Q.FAMILIES[family]
    N = 16
    u0 = np.asarray(Q.U0_NOMINAL[family])[:, None] * np.ones((D, N))
    p = np.asarray(Q.P_NOMINAL[family])
    dWf, Wf = _fine_path(M, N, seed=5)
    at = (TS_CONV / T_CONV * S_FINE).round().astype(int)
    ref = [Q.closed_gradient(family, u0[:, i], p, Wf[at][:, :, i], TS_CONV) for i in range(N)]
    ref_du0, ref_dp = np.array([r[0] for r in ref]).T, np.array([r[1] for r in ref]).T
    errs = []
    for S in S_COARSE:
        dW = dWf.reshape(S, S_FINE // S, M, N).sum(1)
        du0, dp, _ = Q.gradient("f64", family, "euler_heun", sensealg, u0, p, dW, T_CONV / S, TS_CONV)
        errs.append(_err(du0, dp, ref_du0, ref_dp))
    order = _order(errs)
    print(f"{family} {sensealg}: errors {np.array(errs)}, order {order:.2f}")
    assert 0.8 < order < 1.3 and errs[-1] < 5e-3


@pytest.mark.parametrize("sensealg", ["backsolve", "interpolating"])
def test_mixing_gradient_approaches_finite_differences(sensealg):
    fam, N, d = "sde_mixing", 8, 1e-5
    u0 = np.asarray(Q.U0_NOMINAL[fam])[:, None] * np.ones((2, N))
    p = np.asarray(Q.P_NOMINAL[fam])
    pm = np.repeat(p[:, None], N, 1)
    dWf, _ = _fine_path(2, N, seed=6)
    errs = []
    for S in S_COARSE:
        dW, h = dWf.reshape(S, S_FINE // S, 2, N).sum(1), T_CONV / S
        du0, dp, _ = Q.gradient("ld", fam, "euler_heun", sensealg, u0, p, dW, h, TS_CONV)
        L = lambda uu, pp: Q.loss(fam, "euler_heun", uu, pp, dW, h, TS_CONV)
        e_u = [np.eye(2)[:, [j]] * d for j in range(2)]
        e_p = [np.eye(4)[:, [q]] * d for q in range(4)]
        fd_u0 = np.array([(L(u0 + e, pm) - L(u0 - e, pm)) / (2 * d) for e in e_u], dtype=np.float64)
        fd_p = np.array([(L(u0, pm + e) - L(u0, pm - e)) / (2 * d) for e in e_p], dtype=np.float64)
        errs.append(_err(du0, dp, fd_u0, fd_p))
    order = _order(errs)
    print(f"mixing {sensealg}: distance from central differences {np.array(errs)}, order {order:.2f}")
    assert 0.75 < order < 1.4 and errs[-1] < 1e-3


@pytest.mark.parametrize("family", Q.PLUGINS)
def test_long_double_stands_in_for_40_digits(family):
    c = dict(family=family, stepper="euler_heun", sa="interp", cost="vector_dgdp", p="member", noise="regen", saveat="no_T")
    u0, p, cost, dgdp, _ = Q.problem(c, 2, seed=23)
    M = Q.FAMILIES[family][4]
    dW = np.sqrt(R.H) * np.random.default_rng(24).standard_normal((R.S_STEPS, M, 2))
    for sa in ("backsolve", "interpolating"):
        g = [Q.gradient(k, family, "euler_heun", sa, u0, p, dW, R.H, R.SAVEATS["no_T"], cost=cost, dgdp=dgdp) for k in ("ld", "mp")]
        assert R.rel_err(g[0][0], g[1][0]).max() < 1e-15 and R.rel_err(g[0][1], g[1][1]).max() < 1e-15
