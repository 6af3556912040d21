"""The neural-ODE restatement of tests/mlp_restatement.py checked on its own, and the CPU oracle checked against it
(no GPU).

* The hand-written backprop (df/dp)' lam against complex steps of f, in 40 digits (1e-30) and long double (1e-17), on
  parameters from every block: all of b3 and W1, the corners and the diagonal of W2 (a transposed W2 shows there),
  random entries of W2, b1, b2 and W3.
* The long-double restatement against the 40-digit one on one member, the whole gradient of each sensealg with and
  without events (1e-15): long double is then enough for many members.
* InterpolatingAdjoint and GaussAdjoint converge at order about five as dt halves from 0.5 to 1/32 (T = 1.5), a
  relation that does not involve the oracle.
* Separation guards: where a test pins a sensealg at 1e-12, the other sensealg and three wrong kernels restated
  (mirrored Gauss nodes of the forward dense output, a linear dense output, event scales dropped in the reverse pass)
  differ from the correct restatement by at least 1e3 x 1e-12.  At C4's dt = 0.05 they do not (the sensealgs differ by
  1e-12 there), so the dt = 0.05 cases pin the arithmetic, and dt = 0.25 / 0.5 pin the algorithm.
* oracle/adjoint_oracle.c (mlp_hidden = 64) against the long-double restatement over a pairwise matrix of sensealg x
  cost (scalar affine, per-component affine, explicit) x (plain, no_start, events with scales != 1, one of them 0, on
  consecutive grid points, at n = 1 and n = S - 1 and on save times) x dt (0.05 = C4, 0.25, 0.5): du0 per member and
  component floored at 1e-6 of the member's largest, dp per parameter floored at 1e-3 of its block's largest, both at
  1e-12.  The oracle's dp misses a floor of 1e-6 by up to 1e-11 at entries 1e-5 of W2's largest, where its error is
  6e-16 of the block's scale: fp64 rounding, not an algorithmic difference (mlp_restatement.DP_FLOOR).
"""
import os
import sys

import numpy as np
import pytest

import mpmath as mp

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(HERE)
for d in (ROOT, HERE):
    if d not in sys.path:
        sys.path.insert(0, d)

import mlp_restatement as R
import test_gpu_fixed_reference as FR
from oracle import oracle as O

T_END = 1.5
COSTS = {"scalar": (1.0, -0.5), "vector": (np.array([0.7, -1.3]), np.array([0.25, 0.9])), "explicit": "explicit"}


def event_table(S):
    """hybrid-NODE events {n: (scale[2], shift[2])}: n = 1 and 2 (consecutive), n = S - 1, scales distinct per component
    and one of them 0; S = 3 keeps n = 1, 2"""
    ev = {1: (np.array([0.5, 1.5]), np.array([0.2, 0.0])), 2: (np.array([0.0, 1.25]), np.array([-0.1, 0.3])),
          S - 1: (np.array([1.2, 0.8]), np.array([0.0, -0.2]))}
    return {n: v for n, v in ev.items() if 0 < n < S}


def device_events(ev, dt):
    """{n: (s, c)} -> (times, scale[E][2], shift[E][2]) of set_events / make_cfg"""
    ns = sorted(ev)
    return np.array([n * dt for n in ns]), np.array([ev[n][0] for n in ns]), np.array([ev[n][1] for n in ns])


def setup(N, dt, cost, mode, seed=0, T=T_END, saveat=None):
    """-> (restatement problem, saveat, u0, p, dLdu, device events or None); saves at every grid point, t0 included"""
    S = int(round(T / dt))
    rng = np.random.default_rng(seed)
    u0 = rng.uniform(-2, 2, (2, N))
    p = R.weights()
    grid = np.arange(S + 1) * dt
    saveat = grid if saveat is None else saveat
    sos = {int(round(t / dt)): k for k, t in enumerate(saveat)}
    dLdu = rng.standard_normal((len(saveat), 2, N)) if cost == "explicit" else None
    ev = event_table(S) if mode == "events" else None
    pr = R.problem(dt, S, u0, p, sos, COSTS[cost], dLdu, ev, no_start=mode == "no_start")
    return pr, saveat, u0, p, dLdu, None if ev is None else device_events(ev, dt)


def oracle_gradient(sa, cost, mode, dt, saveat, u0, p, dLdu, dev_ev, T=T_END):
    kw = dict(cost=("explicit",) if cost == "explicit" else ("affine", 0.0, 0.0), no_start=mode == "no_start", mlp_hidden=R.H,
              events=dev_ev)
    if cost != "explicit":
        kw["cost_vec"] = COSTS[cost]
    cfg = O.make_cfg("mlp", sa, "tsit5_fixed", u0.shape[1], saveat, 0.0, T, dt=dt, **kw)
    return O.gradient(cfg, saveat, u0, p, dLdu=dLdu)


# pairwise over cost x mode x dt x sensealg (an L9 orthogonal array)
MATRIX = [("scalar", "plain", 0.05, "interpolating"), ("scalar", "no_start", 0.25, "gauss"), ("scalar", "events", 0.5, "interpolating"),
          ("vector", "plain", 0.25, "interpolating"), ("vector", "no_start", 0.5, "interpolating"), ("vector", "events", 0.05, "gauss"),
          ("explicit", "plain", 0.5, "gauss"), ("explicit", "no_start", 0.05, "interpolating"), ("explicit", "events", 0.25, "gauss")]


def label(c):
    return f"{c[3]}-{c[0]}-{c[1]}-dt{c[2]}"


# ------------------------------------------------------------------------------------------------------------------------


def _sample_params(rng):
    W2 = lambda i, j: R.OW2 + j * R.H + i
    q = list(range(R.OB3, R.P)) + list(range(R.OW1, R.OB1))
    q += [W2(0, 0), W2(0, 63), W2(63, 0), W2(63, 63), W2(1, 62), W2(62, 1)] + [W2(i, i) for i in range(0, 64, 7)]
    for blk, n in (("W2", 12), ("b1", 6), ("b2", 6), ("W3", 8)):
        sl = R.BLOCKS[blk]
        q += list(rng.choice(np.arange(sl.start, sl.stop), n, replace=False))
    return sorted(set(int(v) for v in q))


@pytest.mark.parametrize("kind_name,tol", [("mp", 1e-30), ("ld", 1e-17)])
def test_backprop_vjp_matches_complex_steps(kind_name, tol):
    rng = np.random.default_rng(7)
    kind = FR.Kind(kind_name)
    qs = _sample_params(rng)
    M = 2 if kind_name == "mp" else 5
    with (mp.workdps(FR.DPS) if kind_name == "mp" else FR._nullctx()):
        y = [kind.arr(rng.uniform(-2, 2, M)) for _ in range(2)]
        lam = [kind.arr(rng.standard_normal(M)) for _ in range(2)]
        pk = kind.arr(R.weights().reshape(-1, 1))
        g = R.MLP.vjp_p(kind, y, pk, lam)
        yc = [kind.cplx(v) for v in y]
        worst = 0.0
        for q in qs:
            pc = np.array([[v] for v in kind.cplx(pk[:, 0])], dtype=object) if kind_name == "mp" else pk.astype(np.clongdouble)
            pc[q, 0] = pc[q, 0] + kind.idelta
            F = R.MLP(yc, pc)
            cs = kind.imag(sum(lam[c] * F[c] for c in range(2))) / kind.d
            scale = max(max(abs(v) for v in cs), 1e-3 * float(max(abs(v) for v in g.ravel())))
            worst = max(worst, float(max(abs(a - b) for a, b in zip(g[q], cs)) / scale))
        # J' lam of the backprop against the complex step the restatement uses for it
        ju = R.backprop(y, pk, lam)[2]
        jcs = FR.vjp(kind, R.MLP, y, pk, lam, "u")
        worst_u = float(max(abs(ju[c][m] - jcs[c][m]) / abs(jcs[c][m]) for c in range(2) for m in range(M)))
    print(f"{kind_name}: {len(qs)} parameters, largest relative difference {worst:.1e}; J' lam {worst_u:.1e}")
    assert worst <= tol and worst_u <= tol


@pytest.mark.parametrize("sa", ["interpolating", "gauss"])
@pytest.mark.parametrize("mode", ["plain", "events"])
def test_long_double_matches_40_digits(sa, mode):
    """one member, dt = 0.5 (S = 3, events at n = 1 and 2), vector affine cost: 1e-15, dp floored at 1e-3 of its block's
    largest.  Below that floor the long double's own rounding shows (about 1e-19 of the block's scale: 1.4e-15 of a
    W2 entry 1e-4 of W2's largest with events), still 1e-2 of 1e-12 at a floor of 1e-6."""
    pr = setup(1, 0.5, "vector", mode, seed=4)[0]
    a, b = R.restate("mp", pr, sa), R.restate("ld", pr, sa)
    e_u = R.rel_err(b["du0"], a["du0"])
    e_p, e_p6 = R.dp_err(b["mu"].sum(1), a["mu"].sum(1))[0], R.dp_err(b["mu"].sum(1), a["mu"].sum(1), floor=1e-6)[0]
    e_s = np.abs(b["us"] - a["us"]).max() / np.abs(a["us"]).max()
    print(f"{sa} {mode}: long double vs 40 digits: states {e_s:.1e} du0 {e_u:.1e} dp {e_p:.1e} (floored at 1e-6: {e_p6:.1e})")
    assert max(e_s, e_u, e_p) <= 1e-15 and e_p6 <= 1e-14


def test_sensealgs_converge_at_fifth_order():
    dts = [0.5, 0.25, 0.125, 0.0625, 0.03125]
    out = {}
    for sa in ("interpolating", "gauss"):
        res = []
        for dt in dts:
            S = int(round(T_END / dt))
            pr = setup(2, dt, "scalar", "plain", seed=2, saveat=np.array([0.0, 0.5, 1.0, 1.5]))[0]
            r = R.restate("ld", pr, sa)
            res.append(np.concatenate([r["du0"].ravel(), r["mu"].sum(1)]))
        out[sa] = res
    fine = out["gauss"][-1]                                 # the two sensealgs agree to far below the coarse errors
    assert np.abs(out["interpolating"][-1] - fine).max() / np.abs(fine).max() < 1e-9
    for sa, res in out.items():
        err = [np.abs(r - fine).max() / np.abs(fine).max() for r in res[:-1]]
        orders = [np.log2(err[i] / err[i + 1]) for i in range(len(err) - 1)]
        print(f"{sa}: errors {['%.2e' % e for e in err]}, observed orders {['%.2f' % o for o in orders]}")
        assert all(4.0 <= o <= 6.5 for o in orders), (sa, orders)


# where a test pins a sensealg or a variant at 1e-12, the correct restatement differs from the wrong one by >= 1e3 x that
SEPARATION = [("interpolating", "other_sensealg", 0.25), ("interpolating", "other_sensealg", 0.5), ("interpolating", "linear_dense", 0.25),
              ("gauss", "mirrored_gauss_nodes", 0.25), ("gauss", "mirrored_gauss_nodes", 0.5), ("gauss", "linear_dense", 0.5),
              ("interpolating", "no_event_scale", 0.25), ("gauss", "no_event_scale", 0.05)]


def separation(sa, variant, dt, N=4):
    """-> (du0 distance, dp distance per block) of the wrong restatement from the correct one"""
    pr = setup(N, dt, "vector", "events" if variant == "no_event_scale" else "plain", seed=9)[0]
    good = R.restate("ld", pr, sa)
    if variant == "other_sensealg":
        bad = R.restate("ld", pr, "gauss" if sa == "interpolating" else "interpolating")
    else:
        bad = R.restate("ld", pr, sa, variant=variant)
    return R.rel_err(bad["du0"], good["du0"]), R.dp_err(bad["mu"].sum(1), good["mu"].sum(1))[1]


@pytest.mark.parametrize("sa,variant,dt", SEPARATION)
def test_separation_guard(sa, variant, dt):
    e_u, per = separation(sa, variant, dt)
    print(f"{sa} vs {variant} at dt {dt}: du0 {e_u:.1e}, dp by block {({k: float('%.1e' % v) for k, v in per.items()})}")
    # the sensealgs and the mirrored Gauss nodes differ in dp only (du0 is the same state adjoint), in every block but
    # b3 = the integral of lambda, which both quadratures take alike
    assert min(v for k, v in per.items() if k != "b3") >= 1e3 * 1e-12, per
    if variant in ("linear_dense", "no_event_scale"):
        assert e_u >= 1e3 * 1e-12


def test_sensealgs_do_not_separate_at_c4_dt():
    """dt = 0.05: InterpolatingAdjoint and GaussAdjoint differ by less than 1e3 x 1e-12 (why the dt = 0.05 cases do not
    claim to pin the sensealg)"""
    _, per = separation("interpolating", "other_sensealg", 0.05)
    print("dt 0.05, interpolating vs gauss, dp by block:", {k: float('%.1e' % v) for k, v in per.items()})
    assert max(per.values()) < 1e3 * 1e-12


@pytest.mark.parametrize("c", MATRIX, ids=label)
def test_oracle_matches_the_long_double_restatement(c):
    cost, mode, dt, sa = c
    N = 6
    pr, saveat, u0, p, dLdu, dev_ev = setup(N, dt, cost, mode, seed=3)
    ref = R.restate("ld", pr, sa)
    o = oracle_gradient(sa, cost, mode, dt, saveat, u0, p, dLdu, dev_ev)
    e_s = np.abs(o["saved"] - ref["us"]).max() / np.abs(ref["us"]).max()
    e_u = R.rel_err(o["du0"], ref["du0"])
    e_p, per = R.dp_err(o["dp"], ref["mu"].sum(1))
    print(f"{label(c)}: oracle vs long double: saved {e_s:.1e} du0 {e_u:.1e} dp {e_p:.1e} (worst block {max(per, key=per.get)})")
    assert e_s <= 1e-13 and e_u <= 1e-12 and e_p <= 1e-12
