"""Whole gradients of the fixed-step Tsit5 path (csrc/ode_tsit5.cuh, csrc/tsit5_quad.cuh) against a restatement of the
fixed-grid algorithm in 40 digits (mpmath), derivatives by complex steps of the right-hand sides of
tests/ros23_restatement.py (never from families.cuh):

* the forward solve from u0, the tableau as published, events applied between steps;
* the reverse solve with adjoint stage s at y(t_{n+1} - c_s h), y the forward step's own dense output (published
  b_j(theta)), lambda += dg/du at the save times (not at t0 under no_start), lambda *= s and the parameters of the
  segment below at an event;
* dG/dp per sensealg: InterpolatingAdjoint integrates mu with the same tableau; GaussAdjoint with 3-point Gauss-Legendre
  per step, lambda from the adjoint step's own dense output; GaussKronrodAdjoint with the G3/K7 bisection of
  integrate_gk_step (bisect while sum |K - G| >= 1e-7), every decision asserted to lie clear of the threshold;
  QuadratureAdjoint the exact integral of each step's polynomial integrand (8-point Gauss-Legendre, exact to degree 15);
  BacksolveAdjoint the augmented system integrated backwards, its y reset to the forward solution at every step, at
  the save times, or never.

du0 and dp are compared per member and component at 1e-12 relative, the component floored at 1e-6 of the member's
largest (the Rosenbrock23 reference's convention); QuadratureAdjoint at its quadgk tolerance (1e-10); fp32 runs at
2000 eps32, about the rounding a 20-step fp32 solve accumulates.  The CPU oracle's distance from the same reference
is printed beside the device's.  The launch-geometry sweep (S = 1..9 steps, fewer chunks than TMA pipeline stages
below 8; block_threads 32, 96, 160, 224, the last two with a rotating top warp row) compares every member against the
same restatement run in np.longdouble (vectorised over the members; 19 digits are plenty at 1e-12).

Lorenz stays at T <= 0.5, where chaotic growth does not swamp the bound.  C2 at full size is covered step by step by
tests/test_gpu_fixed_probe.py.
"""
import os
import sys
import time
from fractions import Fraction

import numpy as np
import pytest

import mpmath as mp

from ros23_restatement import A_TXT, C_TXT, b_exact, f_lorenz, f_lv, f_robertson

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
if ROOT not in sys.path:
    sys.path.insert(0, ROOT)
DPS = 40
LD = np.longdouble
FAMS = {"lv": (f_lv, 2, 4), "lorenz": (f_lorenz, 3, 3), "robertson": (f_robertson, 3, 3)}
GK_TOL = 1e-7


class Kind:
    """the number type of a restatement run: 'mp' (object arrays of mpf, 40 digits) or 'ld' (np.longdouble arrays)"""

    def __init__(self, name):
        self.name = name
        if name == "mp":
            self.d = mp.mpf("1e-30")
            self.idelta = mp.mpc(0, self.d)
        else:
            self.d = LD("1e-30")
            self.idelta = np.clongdouble(1j) * self.d

    def const(self, x):
        """a Fraction, decimal string or float as a scalar of this kind"""
        fr = Fraction(x)
        if self.name == "mp":
            return mp.mpf(fr.numerator) / fr.denominator
        with mp.workdps(30):
            return LD(mp.nstr(mp.mpf(fr.numerator) / fr.denominator, 25))

    def arr(self, a):
        a = np.asarray(a, dtype=np.float64)
        return np.array([mp.mpf(float(v)) for v in a.ravel()], dtype=object).reshape(a.shape) if self.name == "mp" else a.astype(LD)

    def cplx(self, a):
        return np.array([mp.mpc(v) for v in a], dtype=object) if self.name == "mp" else np.asarray(a, dtype=LD).astype(np.clongdouble)

    def imag(self, z):
        return np.array([mp.im(v) for v in z], dtype=object) if self.name == "mp" else np.asarray(z).imag

    def zeros(self, M):
        return self.arr(np.zeros(M))

    def f64(self, a):
        return np.array([float(v) for v in a]) if self.name == "mp" else np.asarray(a, dtype=np.float64)


def vjp(kind, f, y, p, l, wrt):
    """(df/du)' l (wrt = 'u') or (df/dp)' l (wrt = 'p') by complex steps of l' f(y, p); y, p, l lists of member arrays.
    A family with many parameters supplies (df/dp)' l itself, as f.vjp_p(kind, y, p, l) -> one [P][M] array"""
    if wrt == "p" and hasattr(f, "vjp_p"):
        return f.vjp_p(kind, y, p, l)
    yc, pc = [kind.cplx(v) for v in y], ([kind.cplx(v) for v in p] if wrt == "p" else p)
    out = []
    for c in range(len(y) if wrt == "u" else len(p)):
        yy, pp = list(yc), list(pc)
        if wrt == "u":
            yy[c] = yy[c] + kind.idelta
        else:
            pp[c] = pp[c] + kind.idelta
        out.append(kind.imag(sum(l[r] * v for r, v in enumerate(f(yy, pp)))) / kind.d)
    return out


class Tab:
    def __init__(self, kind):
        self.A = [[kind.const(v) for v in row] for row in A_TXT]
        self.c = [kind.const(v) for v in C_TXT]
        self.kind = kind
        self._b = {}

    def b(self, th):
        """b_j(theta), j = 0..6 (theta a Fraction or float)"""
        key = Fraction(th)
        if key not in self._b:
            self._b[key] = [self.kind.const(b_exact(j, key)) for j in range(7)]
        return self._b[key]


def lin(a, xs, ws):
    """a + sum_j ws[j] xs[j] componentwise (xs: list of states)"""
    return [a[c] + sum(w * x[c] for w, x in zip(ws, xs)) for c in range(len(a))]


def axpy(mu, w, g):
    """mu + w g over the parameters: g a list of member arrays, or one [P][M] array from a family's vjp_p"""
    if isinstance(g, np.ndarray) and g.ndim == 2:
        return np.asarray(mu) + w * g
    return [mu[q] + w * g[q] for q in range(len(mu))]


class Problem:
    """one fixed-grid problem: family (a name of FAMS or a triple (f, D, P)), h, S, u0[D][M], per-member p[P][M], save
    table {n: k}, cost ('explicit' or (a, b), scalars or per-component vectors), events {n: (s, c, ps, pc)}, continuous
    cost (a, b) or None, no_start"""

    def __init__(self, family, h, S, u0, p, sos, cost, dLdu=None, events=None, cont=None, no_start=False):
        self.f, self.D, self.P = FAMS[family] if isinstance(family, str) else family
        self.h, self.S, self.u0, self.p, self.sos, self.cost, self.dLdu = h, S, u0, p, sos, cost, dLdu
        self.events, self.cont, self.no_start = events or {}, cont, no_start


def params_of(kind, pr, n):
    """parameters in force on step n (after the events at grid points <= n)"""
    p = kind.arr(pr.p)
    for m in sorted(pr.events):
        if m > n:
            break
        _, _, ps, pc = pr.events[m]
        if ps is not None:
            p = [kind.const(ps[q]) * p[q] + kind.const(pc[q]) for q in range(pr.P)]
    return p


def forward(kind, tab, pr):
    """-> u[n] (post-event), stages K[n] = [k1..k6, k7 = f(u_{n+1}^-)], p_n"""
    h = kind.const(pr.h)
    u = [kind.arr(v) for v in pr.u0]
    us, Ks, ps = [u], [], []
    for n in range(pr.S):
        p = params_of(kind, pr, n)
        k = [pr.f(u, p)]
        for s in range(1, 7):
            z = lin(u, k, [h * a for a in tab.A[s]])
            if s < 6:
                k.append(pr.f(z, p))
        k.append(pr.f(z, p))
        if n + 1 in pr.events and n + 1 < pr.S:
            sc, sh, _, _ = pr.events[n + 1]
            z = [kind.const(sc[c]) * z[c] + kind.const(sh[c]) for c in range(pr.D)]
        us.append(z)
        Ks.append(k)
        ps.append(p)
        u = z
    return us, Ks, ps


def dense(kind, tab, h, u, k, th):
    """u + h sum_j b_j(theta) k_j"""
    return lin(u, k, [h * w for w in tab.b(th)])


def jump(kind, pr, n, y):
    if n not in pr.sos:
        return None
    if pr.cost == "explicit":
        return [kind.arr(pr.dLdu[pr.sos[n], c]) for c in range(pr.D)]
    a, b = (np.broadcast_to(np.asarray(v, dtype=np.float64), (pr.D,)) for v in pr.cost)
    return [kind.const(a[c]) * y[c] + kind.const(b[c]) for c in range(pr.D)]


def add_cont(kind, pr, y, ka):
    if pr.cont is None:
        return ka
    a, b = pr.cont
    return [ka[c] + kind.const(a) * y[c] + kind.const(b) for c in range(pr.D)]


GL8 = None


def _gl(n):
    """n-point Gauss-Legendre nodes and weights on [0, 1] in 40 digits"""
    with mp.workdps(DPS + 10):
        xs, ws = [], []
        for i in range(1, n + 1):
            x = mp.cos(mp.pi * (i - mp.mpf(1) / 4) / (n + mp.mpf(1) / 2))
            for _ in range(100):
                p0, p1 = mp.mpf(1), x
                for m in range(2, n + 1):
                    p0, p1 = p1, ((2 * m - 1) * x * p1 - (m - 1) * p0) / m
                dp = n * (x * p1 - p0) / (x * x - 1)
                dx = p1 / dp
                x -= dx
                if abs(dx) < mp.mpf(10) ** (-DPS - 5):
                    break
            xs.append((1 - x) / 2)
            ws.append(1 / ((1 - x * x) * dp * dp))
    return xs, ws


def reverse(kind, tab, pr, sensealg, us, Ks, ps, gk_log=None, ckpt_mode="save", gauss_y=None):
    """-> (du0[D][M], dp[P][M]) of the restatement; gauss_y(tha) -> the forward dense output's theta at a Gauss node
    (1 - tha; other maps restate a wrong kernel)"""
    f, D, P = pr.f, pr.D, pr.P
    h = kind.const(pr.h)
    M = len(us[0][0])
    mu = [kind.zeros(M) for _ in range(P)]
    S = pr.S
    if sensealg == "backsolve":
        return _backsolve(kind, tab, pr, us, Ks, ps, ckpt_mode)
    lam = [kind.zeros(M) for _ in range(D)]
    jT = jump(kind, pr, S, us[S])
    if jT is not None:
        lam = lin(lam, [jT], [1])
    for n in range(S - 1, -1, -1):
        p, k, un = ps[n], Ks[n], us[n]
        yend = dense(kind, tab, h, un, k, 1)                 # u_{n+1}^-: the left limit at an event
        ys = [yend] + [dense(kind, tab, h, un, k, 1 - Fraction(C_TXT[s])) for s in range(1, 5)] + [un, un]
        ka, ls = [], []
        for s in range(7):
            l_s = lin(lam, ka, [h * a for a in tab.A[s]]) if s else lam
            ls.append(l_s)
            ka.append(add_cont(kind, pr, ys[s], vjp(kind, f, ys[s], p, l_s, "u")))
        if sensealg == "interpolating":
            for s in range(6):
                g = vjp(kind, f, ys[s], p, ls[s], "p")
                mu = axpy(mu, h * tab.A[6][s], g)
        else:
            def node(tha):
                """integrand at time t_{n+1} - tha h: (df/dp)' lambda, lambda from the adjoint step's dense output"""
                lq = dense(kind, tab, h, lam, ka, tha)
                yq = dense(kind, tab, h, un, k, gauss_y(tha) if gauss_y else 1 - Fraction(tha) if not isinstance(tha, mp.mpf) else 1 - tha)
                return vjp(kind, f, yq, p, lq, "p")
            if sensealg == "gauss":
                a = Fraction(1, 2) * (1 - Fraction(mp.nstr(mp.sqrt(mp.mpf("0.6")), 45)))
                for tha, w in ((a, Fraction(5, 9)), (Fraction(1, 2), Fraction(8, 9)), (1 - a, Fraction(5, 9))):
                    g = node(tha)
                    mu = axpy(mu, h / 2 * kind.const(w), g)
            elif sensealg == "quadrature":
                global GL8
                if GL8 is None:
                    GL8 = _gl(8)
                for x, w in zip(*GL8):
                    g = node(Fraction(mp.nstr(x, 45)))
                    mu = [mu[q] + h * kind.const(mp.nstr(w, 45)) * g[q] for q in range(P)]
            elif sensealg == "gauss_kronrod":
                mu = _gk_step(kind, node, pr.h, mu, P, gk_log)
        lam = ls[6]
        # jump at t_n, then the reverse affect of an event there
        if not (pr.no_start and n == 0):
            j = jump(kind, pr, n, un)
            if j is not None:
                lam = lin(lam, [j], [1])
        if n in pr.events and n > 0:
            sc, _, psc, _ = pr.events[n]
            lam = [kind.const(sc[c]) * lam[c] for c in range(D)]
            if psc is not None:
                mu = [kind.const(psc[q]) * mu[q] for q in range(P)]
    return lam, mu


X7 = ["0.960491268708020283423507092629080", "0.774596669241483377035853079956480", "0.405845151377397166906606412076961"]
W7 = ["0.104656226026467265193823857192073", "0.268488089868333440728569280666710", "0.401397414775962222905051818618432",
      "0.450916538658474142345110087045571"]


def _gk_step(kind, node, h, mu, P, log):
    """integrate_gk_step<P, 3> over local time [h, 0] (theta_a = 1 - s / h): depth first, left half first; every decision
    logged as (err, the fp64-scale magnitude of the sum) per member"""
    xs = [-Fraction(X7[0]), -Fraction(X7[1]), -Fraction(X7[2]), Fraction(0), Fraction(X7[2]), Fraction(X7[1]), Fraction(X7[0])]
    ws = [Fraction(v) for v in W7] + [Fraction(W7[2]), Fraction(W7[1]), Fraction(W7[0])]
    gs = [Fraction(5, 9), Fraction(8, 9), Fraction(5, 9)]
    hF = Fraction(h)
    M = len(mu[0])
    stack = [(hF, Fraction(0), 0, np.ones(M, dtype=bool))]
    while stack:
        l, r, dep, live = stack.pop()
        K = [kind.zeros(M) for _ in range(P)]
        G = [kind.zeros(M) for _ in range(P)]
        for i in range(7):
            s = (r - l) / 2 * xs[i] + (l + r) / 2
            v = node(1 - s / hF)
            K = [K[q] - kind.const(ws[i]) * v[q] for q in range(P)]        # out = -vjp_p
            if i & 1:
                G = [G[q] - kind.const(gs[i // 2]) * v[q] for q in range(P)]
        half = kind.const((r - l) / 2)
        K = [half * x for x in K]
        G = [half * x for x in G]
        err = kind.f64(sum(abs(K[q] - G[q]) for q in range(P)))
        mag = kind.f64(sum(abs(K[q]) + abs(G[q]) for q in range(P)))
        acc = (err < GK_TOL) | (dep >= 30)
        if log is not None:
            log.extend([(e, m) for e, m, lv in zip(err, mag, live) if lv])
        take = acc & live
        mu = [mu[q] + np.where(take, K[q], kind.zeros(M)) for q in range(P)]
        split = (~acc) & live
        if split.any():
            mid = (l + r) / 2
            stack.append((mid, r, dep + 1, split))
            stack.append((l, mid, dep + 1, split))
    return mu


def _backsolve(kind, tab, pr, us, Ks, ps, mode):
    """BacksolveAdjoint: z = [lambda; mu; y] integrated backwards, ky = -f(y), kl = +J' lambda; at t_n the checkpoint
    reset (mode 'every': every step, 'save': at save times, 'none': never), then the jump (no_start does not apply)"""
    f, D, P, S = pr.f, pr.D, pr.P, pr.S
    h = kind.const(pr.h)
    M = len(us[0][0])
    y = list(us[S])
    lam = [kind.zeros(M) for _ in range(D)]
    mu = [kind.zeros(M) for _ in range(P)]
    j = jump(kind, pr, S, y)
    if j is not None:
        lam = lin(lam, [j], [1])
    for n in range(S - 1, -1, -1):
        p = ps[n]
        ky, kl = [], []
        yy, ll = y, lam
        for s in range(7):
            if s:
                yy = lin(y, ky, [h * a for a in tab.A[s]])
                ll = lin(lam, kl, [h * a for a in tab.A[s]])
            ky.append([-v for v in f(yy, p)])
            kl.append(add_cont(kind, pr, yy, vjp(kind, f, yy, p, ll, "u")))
            if s < 6:
                g = vjp(kind, f, yy, p, ll, "p")
                mu = [mu[q] + h * tab.A[6][s] * g[q] for q in range(P)]
        y, lam = yy, ll
        if mode == "every" or (mode == "save" and n in pr.sos):
            y = list(us[n])
        j = jump(kind, pr, n, y)
        if j is not None:
            lam = lin(lam, [j], [1])
        if n in pr.events and n > 0:
            sc, _, psc, _ = pr.events[n]
            lam = [kind.const(sc[c]) * lam[c] for c in range(D)]
            if psc is not None:
                mu = [kind.const(psc[q]) * mu[q] for q in range(P)]
            y = dense(kind, tab, h, us[n - 1], Ks[n - 1], 1)      # y(tau-): the forward step below the event
    return lam, mu


def restate(kind_name, pr, sensealg, gk_log=None, ckpt_mode="save"):
    kind = Kind(kind_name)
    ctx = mp.workdps(DPS) if kind_name == "mp" else _nullctx()
    with ctx:
        tab = Tab(kind)
        us, Ks, ps = forward(kind, tab, pr)
        lam, mu = reverse(kind, tab, pr, sensealg, us, Ks, ps, gk_log, ckpt_mode)
        return np.array([kind.f64(v) for v in lam]), np.array([kind.f64(v) for v in mu])


class _nullctx:
    def __enter__(self):
        return self

    def __exit__(self, *a):
        return False


# ------------------------------------------------------------------------------------------------------------------------


def rel_err(got, ref, floor=1e-6):
    """per member and component: |got - ref| / max(|ref|, floor * the member's largest |ref|); arrays [C][M]"""
    got, ref = np.asarray(got, dtype=np.float64), np.asarray(ref, dtype=np.float64)
    scale = np.maximum(np.abs(ref), floor * np.abs(ref).max(axis=0, keepdims=True))
    scale = np.where(scale > 0, scale, 1e-300)
    return float(np.max(np.abs(got - ref) / scale))


def t5_problem(family, N, shared_p, T=None):
    rng = np.random.default_rng({"lv": 11, "lorenz": 12, "robertson": 13}[family])
    if family == "lv":
        T, u0, p = T or 2.0, np.exp(0.1 * rng.standard_normal((2, N))), np.array([1.5, 1.0, 3.0, 1.0])
    elif family == "lorenz":
        T, u0, p = T or 0.5, np.array([1.0, 0.0, 0.0])[:, None] + 0.1 * rng.standard_normal((3, N)), np.array([10.0, 28.0, 8.0 / 3.0])
    else:
        T, u0, p = T or 2.0, np.repeat(np.array([[1.0], [0.0], [0.0]]), N, 1), np.array([0.4, 30.0, 10.0])
    if not shared_p:
        p = p[:, None] * np.exp(0.05 * rng.standard_normal((len(p), N)))
    return T, u0, p


def _members_p(p, shared_p, N, dtype="f64"):
    a = np.broadcast_to(p[:, None], (len(p), N)) if shared_p else p
    return np.asarray(a, dtype=np.float32 if dtype == "f32" else np.float64).astype(np.float64)


OBS = {}


def run_case(case, kind="mp"):
    """-> dict(dev=(du0, dp), ref=(du0, dp), oracle=(du0, dp) or None, gk_log)"""
    import scimlsensitivity_jl_b200 as b
    from oracle import oracle as O
    fam, sa, shared_p, dt, T = case["family"], case["sensealg"], case.get("shared_p", True), case["dt"], case.get("T")
    N, dtype = case.get("N", 3), case.get("dtype", "f64")
    T, u0, p = t5_problem(fam, N, shared_p, T)
    S = int(round(T / dt))
    grid = np.arange(S + 1) * dt
    saveat = case["saveat"](grid) if "saveat" in case else grid[::2]
    D, P = FAMS[fam][1], FAMS[fam][2]
    cost = case.get("cost", (1.0, -0.5))
    rng = np.random.default_rng(21)
    dLdu = rng.standard_normal((len(saveat), D, N)) if cost == "explicit" else None
    ev = case.get("events")
    no_start, cont, mode = case.get("no_start", False), case.get("cont"), case.get("ckpt", "save")
    kw = dict(shared_p=shared_p, cost=None if cost == "explicit" else b.AffineCost(*cost), no_start=no_start, dtype=dtype,
              checkpoint_every=case.get("C", 1), block_threads=case.get("block", 0), quad_abstol=1e-12, quad_reltol=1e-12,
              checkpointing=mode != "none", ckpt_every_step=mode == "every")
    eng = b.DeviceEnsemble(fam, sa, "tsit5_fixed", N, saveat, (0.0, T), dt, **kw)
    if cont:
        eng.handle.set_continuous_cost(1, *cont)
    if ev:
        eng.set_events(*ev)
    _, status = eng.forward(u0, p)
    assert (np.asarray(status) == 0).all()
    du0, dp = eng.reverse(dLdu)
    du0, dp = np.asarray(du0, dtype=np.float64).copy(), np.asarray(dp, dtype=np.float64).copy()
    eng.close()
    events = None
    if ev:
        times, sc, sh = ev[0], ev[1], ev[2]
        ps, pc = (ev[3], ev[4]) if len(ev) > 3 else (None, None)
        events = {int(round(t / dt)): (sc[e], sh[e], None if ps is None else ps[e], None if pc is None else pc[e]) for e, t in enumerate(times)}
    u0r = np.asarray(u0, dtype=np.float32 if dtype == "f32" else np.float64).astype(np.float64)
    pr = Problem(fam, dt, S, u0r, _members_p(p, shared_p, N, dtype), {int(round(t / dt)): k for k, t in enumerate(saveat)},
                 "explicit" if cost == "explicit" else cost, dLdu, events, cont, no_start)
    log = [] if sa == "gauss_kronrod" else None
    rdu0, rmu = restate(kind, pr, sa, log, mode)
    rdp = rmu.sum(axis=1) if shared_p else rmu
    orc = None
    if dtype == "f64" and case.get("C", 1) == 1:
        ocfg = O.make_cfg(fam, sa, "tsit5_fixed", N, saveat, 0.0, T, dt=dt, cost=("explicit",) if cost == "explicit" else ("affine",) + tuple(cost),
                          shared_p=shared_p, no_start=no_start, checkpointing=mode != "none", ckpt_every_step=mode == "every",
                          quad_abstol=1e-12, quad_reltol=1e-12, cont_cost=cont, events=ev)
        o = O.gradient(ocfg, saveat, u0, p, dLdu=dLdu)
        orc = (o["du0"], o["dp"])
    return dict(dev=(du0, dp), ref=(rdu0, rdp), oracle=orc, gk_log=log, shared_p=shared_p)


def compare(tag, res, tol, floor=1e-6):
    (du0, dp), (rdu0, rdp) = res["dev"], res["ref"]
    dpv, rdpv = (dp.reshape(-1, 1), rdp.reshape(-1, 1)) if res["shared_p"] else (dp, rdp)
    e_u, e_p = rel_err(du0, rdu0, floor), rel_err(dpv, rdpv, floor)
    line = f"{tag}: device du0 {e_u:.1e} dp {e_p:.1e}"
    if res["oracle"] is not None:
        odu0, odp = res["oracle"]
        odpv = odp.reshape(-1, 1) if res["shared_p"] else odp
        line += f"; oracle du0 {rel_err(odu0, rdu0, floor):.1e} dp {rel_err(odpv, rdpv, floor):.1e}"
    OBS[tag] = max(e_u, e_p) / tol
    print(line)
    assert e_u <= tol and e_p <= tol, line


LV_EV = ([0.5, 1.0, 1.5], np.array([[1.2, 0.9], [1.0, 1.1], [0.8, 1.0]]), np.array([[0.1, 0.0], [-0.05, 0.2], [0.0, 0.0]]))
LV_EVP = LV_EV + (np.array([[1.1, 1.0, 0.95, 1.0], [1.0, 1.05, 1.0, 0.9], [0.9, 1.0, 1.0, 1.1]]),
                  np.array([[0.0, 0.1, 0.0, -0.05], [0.02, 0.0, 0.1, 0.0], [0.0, -0.1, 0.0, 0.0]]))

CASES = {
    "lv interpolating affine": dict(family="lv", sensealg="interpolating", dt=0.1),
    "lv gauss per-member p explicit": dict(family="lv", sensealg="gauss", dt=0.1, shared_p=False, cost="explicit"),
    "lv gausskronrod": dict(family="lv", sensealg="gauss_kronrod", dt=0.1),
    "lv gausskronrod dt 0.2 per-member p": dict(family="lv", sensealg="gauss_kronrod", dt=0.2, shared_p=False),
    "lv quadrature": dict(family="lv", sensealg="quadrature", dt=0.1),
    "lv backsolve save": dict(family="lv", sensealg="backsolve", dt=0.1),
    "lv backsolve every": dict(family="lv", sensealg="backsolve", dt=0.1, ckpt="every"),
    "lv backsolve none": dict(family="lv", sensealg="backsolve", dt=0.1, ckpt="none"),
    "lv interpolating no_start continuous": dict(family="lv", sensealg="interpolating", dt=0.1, no_start=True, cont=(0.5, -0.25)),
    "lv gauss continuous per-member p": dict(family="lv", sensealg="gauss", dt=0.1, shared_p=False, cont=(1.0, 0.5)),
    "lorenz interpolating per-member p": dict(family="lorenz", sensealg="interpolating", dt=0.025, shared_p=False),
    "lorenz gauss explicit no_start": dict(family="lorenz", sensealg="gauss", dt=0.025, cost="explicit", no_start=True),
    "robertson gauss": dict(family="robertson", sensealg="gauss", dt=0.05),
    "lv interpolating events": dict(family="lv", sensealg="interpolating", dt=0.1, events=LV_EV),
    "lv gauss events with parameter change": dict(family="lv", sensealg="gauss", dt=0.1, events=LV_EVP, shared_p=False),
    "lv backsolve events with parameter change": dict(family="lv", sensealg="backsolve", dt=0.1, events=LV_EVP),
}
for _C in (2, 3, 7):
    CASES[f"lv interpolating C={_C} S=23"] = dict(family="lv", sensealg="interpolating", dt=0.1, T=2.3, C=_C, block=32)
    CASES[f"lorenz gauss C={_C} S=23 per-member p"] = dict(family="lorenz", sensealg="gauss", dt=0.02, T=0.46, C=_C, shared_p=False, block=32)
FP32 = {f"lv {sa} fp32": dict(family="lv", sensealg=sa, dt=0.1, dtype="f32") for sa in ("interpolating", "gauss", "backsolve")}
FP32["lorenz gauss fp32 C=3"] = dict(family="lorenz", sensealg="gauss", dt=0.025, dtype="f32", C=3, block=32)


@pytest.mark.gpu
@pytest.mark.parametrize("name", list(CASES))
def test_whole_gradient_against_40_digits(name):
    case = CASES[name]
    t0 = time.perf_counter()
    res = run_case(case)
    tol = 1e-10 if case["sensealg"] == "quadrature" else 1e-12       # QuadratureAdjoint: its quadgk tolerance
    compare(name, res, tol)
    if res["gk_log"] is not None:
        # every bisection decision clear of 1e-7 by far more than the device's rounding of err (eps times the magnitudes
        # of K and G) plus its distance from the restatement (1e-12 of them); some bisect at err in [1e-7, 1e-6), which a
        # threshold of 1e-6 would accept instead
        margins = [abs(e - GK_TOL) / (1e-12 * m + 1e-20) for e, m in res["gk_log"]]
        assert min(margins) > 1, (name, min(margins))
        assert sum(GK_TOL <= e < 1e-6 for e, _ in res["gk_log"]) > 0
        print(f"{name}: {len(res['gk_log'])} decisions, {sum(e >= GK_TOL for e, _ in res['gk_log'])} bisections, "
              f"{sum(GK_TOL <= e < 1e-6 for e, _ in res['gk_log'])} with err in [1e-7, 1e-6), smallest margin {min(margins):.2e}")
    print(f"{name}: {time.perf_counter() - t0:.1f} s; largest error / bound so far {max(OBS.values()):.3f}")


@pytest.mark.gpu
@pytest.mark.parametrize("name", list(FP32))
def test_fp32_whole_gradient(name):
    """fp32 kernels against the 40-digit restatement of the same fp32 inputs: 2000 eps32"""
    res = run_case(FP32[name])
    compare(name, res, 2000 * 1.1920928955078125e-07)


@pytest.mark.gpu
@pytest.mark.parametrize("block", [32, 96, 160, 224])
def test_pipeline_and_travelling_warp_edges(block):
    """S = 1..9 steps (fewer TMA chunks than pipeline stages below 8 steps) for block_threads 32, 96, 160, 224 (the last
    two launch whole 128-thread warp rows whose top row travels): every member of three blocks and a partial one
    against the restatement in long double.  The component floor is 1e-3 of the member's largest here: over one to nine
    steps with a single late save some components of du0 and dp cancel to 1e-5 of the largest, and there the rounding
    of their terms (which the CPU oracle shows as well, 2e-11 relative) exceeds 1e-12 of the component"""
    N = 3 * block + 17
    for S in range(1, 10):
        for sa in ("interpolating", "gauss"):
            case = dict(family="lv", sensealg=sa, dt=0.1, T=0.1 * S, N=N, block=block, shared_p=sa == "gauss",
                        saveat=lambda g: g[::2] if len(g) > 2 else g[-1:])
            res = run_case(case, kind="ld")
            compare(f"sweep block={block} S={S} {sa}", res, 1e-12, floor=1e-3)
