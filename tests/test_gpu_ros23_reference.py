"""Rosenbrock23 adjoints against a controller-free 40-digit reference.

With tolerances of 1e30 every step is accepted, the I-controller's factor clamps to q = 0.1 and the next step is h / q:
the step sequence is a pure function of the fp64 arithmetic on t and h (h0 = 1e-6 (T - t0) forward, -1e-4 (T - t0) in
reverse, `tstop_snap`, clipping to the save times and, for Backsolve with checkpoints at every step, to the forward knots).
The reference below takes the same steps with fp64 times and 40-digit states (mpmath), and builds every Rosenbrock23 stage
from the right-hand side alone:

* the right-hand side from `f` alone: its vector-Jacobian products by complex steps of `f`;
* W = I - h d (d rhs / dz) with the Jacobian of the full augmented right-hand side by central differences in 40 digits (the
  right-hand sides are quadratic in z, so the quotient is exact up to rounding) -- never from `jac` / `djac` / `dvjp_p`;
* dT = d rhs / dt by a central difference in t through the forward interpolant (the interval the kernels' lookup at t,
  continuity :right, chooses);
* GaussAdjoint: the midpoint rule of each reverse step; GaussKronrodAdjoint: the per-step G1/K3 bisection of
  `integrate_gk_step` (threshold 1e-7); QuadratureAdjoint: the exact integral of (df/dp)' lambda over the product of the two
  piecewise-quadratic dense outputs (5-point Gauss-Legendre on every piece between forward and reverse knots).

Compared per member and per component, for LV, Lorenz and Robertson with shared and per-member p: Gauss, GaussKronrod,
Quadrature, Interpolating, Backsolve with and without checkpoints at every step (not Backsolve on Robertson: it blows up
backwards), the LvClone plug-in, the forward step counts and, for QuadratureAdjoint, the reverse step counts.

Under the controller (tolerance 1e-5, forward and reverse) the reference also restates the error estimate (the k3 stage,
the weighted RMS norm over all components of z) and the I-controller, with accept/reject decisions and q on the fp64 value of
the estimate; every decision is asserted to lie more than 1e-6 from EEst = 1, so fp64 and 40 digits take the same steps.
This sees what the accepted-always runs cannot: the error estimate and, through it, every step size and rejection.

Bounds, relative to the component (floored at 1e-6 of the member's largest component): 1e-12.  Robertson: the smaller of
1e-12 (1e-11 under the controller) and the a-priori ceiling 8 cond(W) eps, cond(W) the largest infinity-norm condition
number of the W the reference factors in that run (the probe module shows the LU solve itself within cond(W) eps): 1e-12
with all steps accepted (cond(W) <= 2e4), 5.9e-12 under the controller (cond(W) 3.3e3).  QuadratureAdjoint's dp is compared on the scale of the member's dp vector, the norm its quadgk
stops on.  Observed on an H100 SXM (700 W), all step counts equal: LV <= 2.1e-13, Lorenz <= 7.0e-14, Robertson <= 1.6e-14
(CPU oracle: 2.2e-13, 7.1e-14, 1.6e-14); under the controller LV <= 2.4e-14,
Lorenz <= 4.2e-15, Robertson <= 3.8e-13 (CPU oracle: 8.1e-15, 4.9e-15, 1.6e-12).

The time derivative of InterpolatingAdjoint's mu rows cancels from the Rosenbrock23 step altogether (solution and error
estimate); `test_mu_row_time_derivative_cancels_from_interpolating_steps` shows it on the reference.  Lorenz Backsolve with checkpoints at every
step is not compared: with 1e30 tolerances its last forward step spans 0.44 of [0, 0.5], and y integrated backwards over it
loses 13 digits (the restatement itself moves in the 7th digit between 20 and 40 digits).  The 40-digit reference takes
~55 s of host time, GaussKronrod's bisection and the Robertson runs under the controller most of it."""
import functools

import numpy as np
import pytest

import mpmath as mp

from ros23_restatement import EPS100, f_lorenz, f_lv, f_robertson, problem, register_lv_clone, tstop_snap, vjp_p, vjp_u

ROS_D = 0.29289321881345247559915563789515
DPS = 40
HUGE = 1e30                 # tolerances at which every step is accepted
COST_A, COST_B = 1.0, -0.5
FAM = {"lv": (f_lv, 2, 4), "lv_clone": (f_lv, 2, 4), "lorenz": (f_lorenz, 3, 3), "robertson": (f_robertson, 3, 3)}


def step_factor(eest):
    """the I-controller (exponent 1/3, gamma 0.9, q in [0.1, 5]) on the fp64 value of the error estimate"""
    return max(0.1, min(5.0, max(float(eest), 1e-300) ** (1.0 / 3.0) / 0.9))


ROS_E32 = 6.0 + 1.4142135623730951            # as the kernels fold it


def _eest(h, k1, k2, k3, x, xn, tol):
    """sqrt(mean((h/6 (k1 - 2 k2 + k3) / (tol + tol max(|x|, |xn|)))^2)) in 40 digits"""
    e2 = 0
    for c in range(len(x)):
        e = h / 6 * (k1[c] - 2 * k2[c] + k3[c])
        sc = tol + tol * max(abs(x[c]), abs(xn[c]))
        e2 += (e / sc) ** 2
    return mp.sqrt(e2 / len(x))


# ------------------------------------------------------------------------------------------------------------------------
# 40-digit linear algebra and complex steps


def _solve(W, b):
    return list(mp.lu_solve(W, mp.matrix(b)))


def _cond(W):
    return float(mp.mnorm(W, mp.inf) * mp.mnorm(W ** -1, mp.inf))


def _jac_cs(f, z):
    """df / dz of a plain polynomial f by complex steps: column c = Im f(z + i delta e_c) / delta"""
    L, dl = len(z), mp.mpf("1e-30")
    A = mp.matrix(L, L)
    for c in range(L):
        zc = [mp.mpc(v) for v in z]
        zc[c] += mp.mpc(0, dl)
        col = f(zc)
        for r in range(L):
            A[r, c] = mp.im(col[r]) / dl
    return A


def _jac_cd(rhs, z):
    """d rhs / dz of the augmented right-hand side (which itself holds complex-step VJPs) by central differences in 40
    digits: the right-hand sides are quadratic in z, so the difference quotient is exact up to rounding"""
    L = len(z)
    A = mp.matrix(L, L)
    for c in range(L):
        dl = mp.mpf("1e-12") * max(1, abs(z[c]))
        zp, zm = list(z), list(z)
        zp[c] += dl
        zm[c] -= dl
        fp, fm = rhs(zp), rhs(zm)
        for r in range(L):
            A[r, c] = (fp[r] - fm[r]) / (2 * dl)
    return A


# ------------------------------------------------------------------------------------------------------------------------
# forward solve and its dense output


class Forward:
    """fp64 knots, 40-digit states and stage vectors of the Rosenbrock23 forward solve (autonomous: dT = 0)"""

    def __init__(self, f, u0, p, t0, T, tol):
        D = len(u0)
        self.f, self.p = f, p
        u = [mp.mpf(float(v)) for v in u0]
        self.ft, self.fu, self.k1, self.k2, self.conds = [t0], [u], [], [], []
        self.margin, self.rejects = mp.inf, 0           # closest |EEst - 1| of any accept/reject decision
        t, h = t0, 1e-6 * (T - t0)
        while t < T:
            last = False
            if t + h >= T or abs(t + h - T) < 100 * 2.22e-16 * abs(T):
                h, last = T - t, True
            J = _jac_cs(lambda z: f(z, p), u)
            W = mp.eye(D) - h * ROS_D * J
            self.conds.append(_cond(W))
            f0 = f(u, p)
            k1 = _solve(W, f0)
            f1 = f([u[j] + 0.5 * h * k1[j] for j in range(D)], p)
            k2 = _solve(W, [f1[j] - k1[j] for j in range(D)])
            k2 = [k2[j] + k1[j] for j in range(D)]
            un = [u[j] + h * k2[j] for j in range(D)]
            fn = f(un, p)
            k3 = _solve(W, [fn[j] - ROS_E32 * (k2[j] - f1[j]) - 2 * (k1[j] - f0[j]) for j in range(D)])
            eest = _eest(h, k1, k2, k3, u, un, tol)
            self.margin = min(self.margin, abs(eest - 1))
            q = step_factor(eest)
            if eest > 1:
                self.rejects += 1
                h = h / q
                continue
            tn = T if last else t + h
            self.k1.append(k1)
            self.k2.append(k2)
            self.fu.append(un)
            self.ft.append(tn)
            u, t = un, tn
            h = h / q
        self.n = len(self.ft) - 1

    def interval(self, t, right):
        n, ft = self.n, self.ft
        if right:
            iv = max([k for k in range(n) if ft[k] <= t], default=0)
        else:
            iv = max([k for k in range(n) if k == 0 or ft[k] < t], default=0)
        return min(max(iv, 0), n - 1)

    def eval(self, t, right=True, iv=None):
        """y(t) on the interval the lookup chooses, or on interval iv (a difference in t on a fixed interval)"""
        if iv is None:
            iv = self.interval(t, right)
        ta, h = self.ft[iv], self.ft[iv + 1] - self.ft[iv]
        th = (t - ta) / h if h != 0.0 else mp.mpf(1)
        c1 = th * (1 - th) / (1 - 2 * mp.mpf(ROS_D))
        c2 = th * (th - 2 * mp.mpf(ROS_D)) / (1 - 2 * mp.mpf(ROS_D))
        return [self.fu[iv][j] + h * (c1 * self.k1[iv][j] + c2 * self.k2[iv][j]) for j in range(len(self.fu[iv]))]


# ------------------------------------------------------------------------------------------------------------------------
# reverse solve


def _gl5():
    x, w = np.polynomial.legendre.leggauss(5)
    return [mp.mpf(float(v)) for v in x], [mp.mpf(float(v)) for v in w]


def reverse(sensealg, f, fwd, p, saveat, t0, T, every, tol, drop_mu_dt=False):
    """-> (du0[D], dp[P], nrev, max cond(W), closest |EEst - 1|, rejected steps) of one member"""
    D, P = len(fwd.fu[0]), len(p)
    aug = sensealg in ("interpolating", "backsolve")
    L = (D + P if sensealg == "interpolating" else 2 * D + P) if aug else D
    YO = D + P
    z = [mp.mpf(0)] * L
    if sensealg == "backsolve":
        z[YO:YO + D] = list(fwd.fu[fwd.n])

    def rhs(tt, x, iv=None):
        y = x[YO:YO + D] if sensealg == "backsolve" else fwd.eval(tt, True, iv)
        out = [-v for v in vjp_u(f, y, p, x[:D])]
        if aug:
            out += [-v for v in vjp_p(f, y, p, x[:D])]
        if sensealg == "backsolve":
            out += f(y, p)
        return out

    K = len(saveat)
    state = {"cur": K - 1, "ck": fwd.n}

    def ckpt_if_at(tt):
        if sensealg != "backsolve":
            return
        tol = EPS100 * max(abs(tt), 1.0)
        if every:
            while state["ck"] >= 0 and fwd.ft[state["ck"]] > tt + tol:
                state["ck"] -= 1
            if state["ck"] >= 0 and abs(fwd.ft[state["ck"]] - tt) <= tol:
                z[YO:YO + D] = list(fwd.fu[state["ck"]])
        elif state["cur"] >= 0 and abs(saveat[state["cur"]] - tt) <= tol:
            z[YO:YO + D] = fwd.eval(saveat[state["cur"]], True)

    def jump_if_at(tt):
        while state["cur"] >= 0 and abs(saveat[state["cur"]] - tt) <= EPS100 * max(abs(tt), 1.0):
            y = z[YO:YO + D] if sensealg == "backsolve" else fwd.eval(saveat[state["cur"]], True)
            for j in range(D):
                z[j] += COST_A * y[j] + COST_B
            state["cur"] -= 1

    acc = [mp.mpf(0)] * P
    recs = []                      # QuadratureAdjoint: (t, hs, z, k1, k2) of every reverse step
    conds = []
    margin, rejects = mp.inf, 0
    t = T
    ckpt_if_at(t)
    jump_if_at(t)
    h = -1e-4 * (T - t0)
    while t > t0:
        cur = state["cur"]
        tstop = t0
        if cur >= 0 and t > saveat[cur] > tstop:
            tstop = saveat[cur]
        if sensealg == "backsolve" and every:
            c2 = state["ck"]
            while c2 >= 0 and fwd.ft[c2] >= t - EPS100 * max(abs(t), 1.0):
                c2 -= 1
            if c2 >= 0 and fwd.ft[c2] > tstop:
                tstop = fwd.ft[c2]
        tn = tstop_snap(t + h, tstop)
        if tn < tstop:
            tn = tstop
        hs = tn - t
        iv = None if sensealg == "backsolve" else fwd.interval(t, True)
        f0 = rhs(t, z)
        A = _jac_cd(lambda x: rhs(t, x, iv), z)
        if sensealg == "backsolve":
            dT = [mp.mpf(0)] * L
        else:          # through the forward interpolant of the interval the lookup at t chooses
            dl = mp.mpf("1e-12") * max(1, abs(t))
            rp, rm = rhs(mp.mpf(t) + dl, z, iv), rhs(mp.mpf(t) - dl, z, iv)
            dT = [(rp[c] - rm[c]) / (2 * dl) for c in range(L)]
            if drop_mu_dt:
                dT[D:D + P] = [mp.mpf(0)] * P
        hd = hs * mp.mpf(ROS_D)
        W = mp.eye(L) - hd * A
        conds.append(_cond(W))
        k1 = _solve(W, [f0[c] + hd * dT[c] for c in range(L)])
        f1 = rhs(t + 0.5 * hs, [z[c] + 0.5 * hs * k1[c] for c in range(L)])
        k2 = _solve(W, [f1[c] - k1[c] for c in range(L)])
        k2 = [k2[c] + k1[c] for c in range(L)]
        zn = [z[c] + hs * k2[c] for c in range(L)]
        fnr = rhs(t + hs, zn)
        k3 = _solve(W, [fnr[c] - ROS_E32 * (k2[c] - f1[c]) - 2 * (k1[c] - f0[c]) + hd * dT[c] for c in range(L)])
        eest = _eest(hs, k1, k2, k3, z, zn, tol)
        margin = min(margin, abs(eest - 1))
        q = step_factor(eest)
        if eest > 1:
            rejects += 1
            h = hs / q
            continue

        def lam(tj):
            th = (tj - t) / hs
            c1 = th * (1 - th) / (1 - 2 * mp.mpf(ROS_D))
            c2 = th * (th - 2 * mp.mpf(ROS_D)) / (1 - 2 * mp.mpf(ROS_D))
            return [z[j] + hs * (c1 * k1[j] + c2 * k2[j]) for j in range(D)]

        def node(tj):
            return [-v for v in vjp_p(f, fwd.eval(tj, False), p, lam(tj))]

        if sensealg == "gauss":
            tj = 0.5 * (tn + t)
            g = node(tj)
            acc = [acc[q] + (0.5 * (tn - t)) * 2 * g[q] for q in range(P)]
        elif sensealg == "gauss_kronrod":
            acc = [acc[q] + v for q, v in enumerate(_gk_step(lambda tj: _node64(f, fwd, p, lam(tj), tj), t, tn, P))]
        elif sensealg == "quadrature":
            recs.append((t, hs, list(z), k1, k2))
        z = zn
        t = tn
        ckpt_if_at(t)
        jump_if_at(t)
        h = hs / q
    if aug:
        return z[:D], z[D:D + P], None, max(conds), margin, rejects
    if sensealg == "quadrature":
        acc = _quad_exact(f, fwd, p, recs, t0, T, D, P)
    return z[:D], acc, len(recs) if sensealg == "quadrature" else None, max(conds), margin, rejects


def _node64(f, fwd, p, lam, tj):
    """-(df/dp)' lambda at a node in fp64 (complex steps of f): the G1/K3 bisection evaluates many nodes, and its decisions
    are taken on fp64 values as in the kernel"""
    y = [complex(float(v)) for v in fwd.eval(tj, False)]
    lf = [float(v) for v in lam]
    out = []
    for q in range(len(p)):
        pc = [complex(float(v)) for v in p]
        pc[q] += 1e-60j
        out.append(-sum(lf[r] * complex(v) for r, v in enumerate(f(y, pc))).imag / 1e-60)
    return out


X3 = [-0.774596669241483377035853079956480, 0.0, 0.774596669241483377035853079956480]
G3 = [0.555555555555555555555555555555556, 0.888888888888888888888888888888889, 0.555555555555555555555555555555556]


def _gk_step(node, bl, br, P):
    """integrate_gk_step<P, 1>: K3 against the midpoint rule, bisect while sum |K - G| >= 1e-7 (depth < 30); fp64 nodes"""
    out = [mp.mpf(0)] * P
    stack = [(bl, br, 0)]
    while stack:
        l, r, dep = stack.pop()
        K, G = [0.0] * P, [0.0] * P
        for i in range(3):
            v = node(0.5 * (r - l) * X3[i] + 0.5 * (l + r))
            K = [K[q] + G3[i] * v[q] for q in range(P)]
            if i == 1:
                G = [G[q] + 2 * v[q] for q in range(P)]
        K = [v * (0.5 * (r - l)) for v in K]
        G = [v * (0.5 * (r - l)) for v in G]
        if sum(abs(K[q] - G[q]) for q in range(P)) < 1e-7 or dep >= 30:
            out = [out[q] + mp.mpf(K[q]) for q in range(P)]
        else:
            mid = 0.5 * (l + r)
            stack += [(mid, r, dep + 1), (l, mid, dep + 1)]
    return out


def _quad_exact(f, fwd, p, recs, t0, T, D, P):
    """int_{t0}^{T} (df/dp)(y(t))' lambda(t) dt over the piecewise quadratics: 5-point Gauss-Legendre on every piece between
    the forward knots and the reverse step ends (exact for the degree-6 integrands)"""
    x, w = _gl5()
    cuts = sorted(set([float(v) for v in fwd.ft] + [r[0] for r in recs] + [r[0] + r[1] for r in recs] + [t0, T]))
    total = [mp.mpf(0)] * P
    for a, b in zip(cuts[:-1], cuts[1:]):
        if b <= a:
            continue
        mid = 0.5 * (a + b)
        iv = fwd.interval(mid, True)
        rec = next(r for r in recs if r[0] + r[1] <= mid <= r[0])        # the reverse step covering the piece
        ts, hs, z, k1, k2 = rec
        A, B = mp.mpf(a), mp.mpf(b)
        for xi, wi in zip(x, w):
            tj = (B - A) / 2 * xi + (A + B) / 2
            th = (tj - ts) / hs
            c1 = th * (1 - th) / (1 - 2 * mp.mpf(ROS_D))
            c2 = th * (th - 2 * mp.mpf(ROS_D)) / (1 - 2 * mp.mpf(ROS_D))
            lam = [z[j] + hs * (c1 * k1[j] + c2 * k2[j]) for j in range(D)]
            g = vjp_p(f, fwd.eval(tj, True, iv), p, lam)
            total = [total[q] + (B - A) / 2 * wi * g[q] for q in range(P)]
    return total


@functools.lru_cache(maxsize=None)
def reference(family, sensealg, shared_p, every, N, tol=HUGE, drop_mu_dt=False):
    """-> dict(du0[D][N], dp[P] or [P][N], fsteps[N], rsteps[N] or None, cond = max cond(W) seen, margin = closest |EEst - 1|
    of any accept/reject decision, rejects = rejected steps, forward and reverse)"""
    f, D, P = FAM[family]
    t0, T, saveat, u0, p = problem(family, N, shared_p)
    du0, dp, fs, rs, cond = np.zeros((D, N)), np.zeros((P, N)), np.zeros(N, np.int32), np.zeros(N, np.int32), 0.0
    margin, rejects = mp.inf, 0
    with mp.workdps(DPS):
        for i in range(N):
            pi = [mp.mpf(float(v)) for v in (p if shared_p else p[:, i])]
            fwd = Forward(f, u0[:, i], pi, t0, T, tol)
            a, b, nrev, c, m, rj = reverse(sensealg, f, fwd, pi, list(saveat), t0, T, every, tol, drop_mu_dt)
            margin, rejects = min(margin, m, fwd.margin), rejects + rj + fwd.rejects
            du0[:, i] = [float(v) for v in a]
            dp[:, i] = [float(v) for v in b]
            fs[i], rs[i] = fwd.n, nrev if nrev is not None else -1
            cond = max(cond, c, max(fwd.conds))
    return {"du0": du0, "dp": dp.sum(axis=1) if shared_p else dp, "fsteps": fs, "rsteps": rs if sensealg == "quadrature" else None,
            "cond": cond, "margin": float(margin), "rejects": rejects, "saveat": saveat, "u0": u0, "p": p, "t": (t0, T)}


def _bound(family, cond, tol=HUGE):
    """1e-12; Robertson: the smaller of its a-priori ceiling 8 cond(W) eps and 1e-12 (1e-11 under the controller)"""
    if family != "robertson":
        return 1e-12
    return min(1e-11 if tol != HUGE else 1e-12, 8 * cond * np.finfo(float).eps)


def _errs(x, ref, floor=1e-6):
    """relative error per component, the denominator floored at `floor` times the member's largest component"""
    x, ref = np.atleast_2d(np.asarray(x, dtype=float).T).T, np.atleast_2d(np.asarray(ref, dtype=float).T).T
    floor = floor * np.abs(ref).max(axis=0, keepdims=True)
    return np.abs(x - ref) / np.maximum(np.abs(ref), np.maximum(floor, 1e-300))


def _dp_floor(sensealg):
    """QuadratureAdjoint's quadgk stops on the norm of the member's dp vector: its components are compared on that scale"""
    return 1.0 if sensealg == "quadrature" else 1e-6


N_MEMBERS = 2
CASES = [(fam, sa, ev) for fam in ("lv", "lorenz", "robertson")
         for sa, ev in (("gauss", False), ("gauss_kronrod", False), ("quadrature", False), ("interpolating", False),
                        ("backsolve", False), ("backsolve", True))
         if not (fam == "robertson" and sa == "backsolve") and not (fam == "lorenz" and ev)] + [("lv_clone", "gauss", False), ("lv_clone", "interpolating", False)]
QUAD_TOL = 1e-13
# under the controller (tolerance 1e-5 forward and reverse): the error estimate, with its k3 stage, sets every step size and
# rejects steps (12 to 174 per case), so a wrong k3 or dT of the lambda rows moves the gradient
CTRL_TOL = 1e-5
CTRL_CASES = [("lv", "interpolating"), ("lorenz", "interpolating"), ("robertson", "interpolating"), ("lv", "gauss"),
              ("robertson", "gauss"), ("lv", "backsolve")]


def _oracle_family(family):
    return "lv" if family == "lv_clone" else family


@pytest.mark.parametrize("family,sensealg,every", [c for c in CASES if c[0] != "lv_clone"])
def test_oracle_matches_the_controller_free_reference(family, sensealg, every):
    """No GPU: the oracle's ros23_step-based gradient at tolerances 1e30 against the reference (pins the oracle's hand-written
    djac / dpjac as a side effect)."""
    from oracle import oracle as O
    for shared_p in (False, True):
        ref = reference(family, sensealg, shared_p, every, N_MEMBERS)
        t0, T = ref["t"]
        cfg = O.make_cfg(family, sensealg, "rosenbrock23", N_MEMBERS, ref["saveat"], t0, T, abstol=1e30, reltol=1e30,
                         cost=("affine", COST_A, COST_B), shared_p=shared_p, ckpt_every_step=every, quad_abstol=QUAD_TOL, quad_reltol=QUAD_TOL)
        got = O.gradient(cfg, ref["saveat"], ref["u0"], ref["p"])
        assert np.array_equal(got["steps"], ref["fsteps"])
        bound = _bound(family, ref["cond"])
        e_u, e_p = _errs(got["du0"], ref["du0"]).max(), _errs(got["dp"], ref["dp"], _dp_floor(sensealg)).max()
        print(f"oracle {family} {sensealg} every={every} shared={shared_p}: du0 {e_u:.1e} dp {e_p:.1e} (bound {bound:.1e}, cond {ref['cond']:.1e})")
        assert e_u <= bound and e_p <= bound, (e_u, e_p, bound)


@pytest.fixture(scope="module")
def lv_clone_registered():
    return register_lv_clone()


@pytest.mark.gpu
@pytest.mark.parametrize("shared_p", [False, True])
@pytest.mark.parametrize("family,sensealg,every", CASES)
def test_device_matches_the_controller_free_reference(lv_clone_registered, family, sensealg, every, shared_p):
    import scimlsensitivity_jl_b200 as b
    ref = reference(family, sensealg, shared_p, every, N_MEMBERS)
    t0, T = ref["t"]
    eng = b.DeviceEnsemble(family, sensealg, "rosenbrock23", N_MEMBERS, ref["saveat"], (t0, T), 0.0, shared_p=shared_p,
                           cost=b.AffineCost(COST_A, COST_B), ckpt_every_step=every, abstol=1e30, reltol=1e30,
                           quad_abstol=QUAD_TOL, quad_reltol=QUAD_TOL)
    eng.handle.set_tolerances(1e30, 1e30, QUAD_TOL, QUAD_TOL)
    saved, status = eng.forward(ref["u0"], ref["p"])
    assert (np.asarray(status) == 0).all()
    du0, dp = eng.reverse()
    fs, rs = eng.step_counts()
    eng.close()
    assert np.array_equal(fs, ref["fsteps"]), (fs, ref["fsteps"])
    if sensealg == "quadrature":
        assert np.array_equal(rs, ref["rsteps"]), (rs, ref["rsteps"])
    bound = _bound(family, ref["cond"])
    e_u, e_p = _errs(du0, ref["du0"]), _errs(dp, ref["dp"], _dp_floor(sensealg))
    print(f"device {family} {sensealg} every={every} shared={shared_p}: du0 {e_u.max():.1e} dp {e_p.max():.1e} "
          f"(bound {bound:.1e}, cond {ref['cond']:.1e}, steps {list(fs)})")
    assert e_u.max() <= bound and e_p.max() <= bound, (e_u, e_p, bound)


@pytest.mark.parametrize("family,sensealg", CTRL_CASES)
def test_oracle_matches_the_reference_under_the_controller(family, sensealg):
    """No GPU: the oracle at tolerance 1e-5 against the reference that restates the error estimate and the I-controller."""
    from oracle import oracle as O
    ref = reference(family, sensealg, False, False, N_MEMBERS, CTRL_TOL)
    assert ref["rejects"] > 0 and ref["margin"] > 1e-6      # decisions far from EEst = 1: fp64 and 40 digits take the same ones
    t0, T = ref["t"]
    cfg = O.make_cfg(family, sensealg, "rosenbrock23", N_MEMBERS, ref["saveat"], t0, T, abstol=CTRL_TOL, reltol=CTRL_TOL,
                     cost=("affine", COST_A, COST_B), shared_p=False)
    got = O.gradient(cfg, ref["saveat"], ref["u0"], ref["p"])
    assert np.array_equal(got["steps"], ref["fsteps"])
    bound = _bound(family, ref["cond"], CTRL_TOL)
    e_u, e_p = _errs(got["du0"], ref["du0"]).max(), _errs(got["dp"], ref["dp"]).max()
    print(f"oracle {family} {sensealg} tol {CTRL_TOL}: du0 {e_u:.1e} dp {e_p:.1e} (bound {bound:.1e}, rejects {ref['rejects']})")
    assert e_u <= bound and e_p <= bound, (e_u, e_p, bound)


@pytest.mark.gpu
@pytest.mark.parametrize("family,sensealg", CTRL_CASES)
def test_device_matches_the_reference_under_the_controller(family, sensealg):
    import scimlsensitivity_jl_b200 as b
    ref = reference(family, sensealg, False, False, N_MEMBERS, CTRL_TOL)
    t0, T = ref["t"]
    eng = b.DeviceEnsemble(family, sensealg, "rosenbrock23", N_MEMBERS, ref["saveat"], (t0, T), 0.0, shared_p=False,
                           cost=b.AffineCost(COST_A, COST_B), abstol=CTRL_TOL, reltol=CTRL_TOL)
    saved, status = eng.forward(ref["u0"], ref["p"])
    assert (np.asarray(status) == 0).all()
    du0, dp = eng.reverse()
    fs, _ = eng.step_counts()
    eng.close()
    assert np.array_equal(fs, ref["fsteps"]), (fs, ref["fsteps"])
    bound = _bound(family, ref["cond"], CTRL_TOL)
    e_u, e_p = _errs(du0, ref["du0"]), _errs(dp, ref["dp"])
    print(f"device {family} {sensealg} tol {CTRL_TOL}: du0 {e_u.max():.1e} dp {e_p.max():.1e} (bound {bound:.1e}, rejects {ref['rejects']})")
    assert e_u.max() <= bound and e_p.max() <= bound, (e_u, e_p, bound)


@pytest.mark.parametrize("family", ["lv", "robertson"])
def test_mu_row_time_derivative_cancels_from_interpolating_steps(family):
    """InterpolatingAdjoint's mu rows have W = [.., I]: hd dT_mu enters k1_mu and k3_mu only, and cancels from both the
    solution (k2_mu = f1_mu - hd F'x_lam, free of k1_mu) and the error estimate (k1_mu - 2 k2_mu + k3_mu: +hd dT_mu from k1,
    -2 hd dT_mu + hd dT_mu from k3).  So ros23_reverse_kernel's dT[D + q] has no effect beyond rounding, and no test of
    its outputs can see it; the 40-digit reference shows the cancellation, under the controller, to fp64 rounding."""
    a = reference(family, "interpolating", False, False, N_MEMBERS, CTRL_TOL)
    with_zero = reference(family, "interpolating", False, False, N_MEMBERS, CTRL_TOL, drop_mu_dt=True)
    assert np.array_equal(a["fsteps"], with_zero["fsteps"]) and a["rejects"] == with_zero["rejects"]
    assert _errs(with_zero["du0"], a["du0"]).max() <= 1e-15 and _errs(with_zero["dp"], a["dp"]).max() <= 1e-15
