"""The general-noise SDE path (csrc/sde_em.cuh with a B200ADJ_FAMILY_SDE_GENERAL family) restated in plain Python, generic
over the number type like tests/sde_restatement.py, whose number kinds, complex-step VJPs, Philox increments and save tables
it reuses.  The model inputs are the drift f and the full D x M diffusion matrix G of the reference's test problems; every
derivative of G comes from complex steps of the contraction l' G(y, p) w, never from examples/sde_noise_families.cuh.

* The forward pass: Euler-Maruyama u + h f + G dW and EulerHeun u + h (f + f~)/2 + (G + G~)/2 dW on the dt grid.
* The reverse pass of SDEAdjointProblem with the (2n + P) x m noise matrix (src/backsolve_adjoint.jl:399-411,
  src/interpolating_adjoint.jl:453-613), stepping dt = -h with the increment w = -dW_{n-1}: the diffusion increment of
  lam is -(dG w/du)' lam, of mu -(dG w/dp)' lam and of y G w -- jacNoise! with noisemixing = true
  (src/derivative_wrappers.jl:1197-1258).  Callbacks, checkpoint modes and no_start as in sde_restatement.reverse.
* EM + BacksolveAdjoint, which the device refuses for general noise, is restated with the reference's transformed drift
  f - J_{vec G}' vec G (src/sde_tools.jl:29-66): for diagonal noise that does not mix it is the Ito correction, which is
  what lets the diagonal families written in the general shape reproduce sde_restatement over its whole matrix.
* Closed forms of the gradients along one Brownian path for the families that have one (Stratonovich solutions).
"""

import itertools

import numpy as np

import mpmath as mp

import sde_restatement as R


# ---- the test problems: drift f(u, p) -> [D], diffusion G(u, p) -> [D][M] -------------------------------------------

def f_roessler(u, p):
    """test/SDE2/sde_nondiag_stratonovich.jl:28-80: f = A u, A = [p1 p2; p2 p1] (1-based there)"""
    return [p[0] * u[0] + p[1] * u[1], p[1] * u[0] + p[0] * u[1]]


def G_roessler(u, p):
    """G[:, j] = B u for both columns, B = [p3 p4; p4 p3]"""
    c0, c1 = p[2] * u[0] + p[3] * u[1], p[3] * u[0] + p[2] * u[1]
    return [[c0, c0], [c1, c1]]


def G_mixing(u, p):
    """:290-322: diag(g) with g1 = g2 = p3 u1 + p4 u2"""
    c = p[2] * u[0] + p[3] * u[1]
    z = c * 0
    return [[c, z], [z, c]]


def f_additive(u, p):
    """:793-822: f = -u"""
    return [-u[0], -u[1]]


def G_additive(u, p):
    """G = [K_R 0; K_I 0], p = [K_R, K_I]"""
    z = p[0] * 0
    return [[p[0], z], [p[1], z]]


def f_nonsquare(u, p):
    """:863-885: f = p1 u, d = 3"""
    return [p[0] * u[0], p[0] * u[1], p[0] * u[2]]


def G_nonsquare(u, p):
    """[diag(p2 u1, p2 u2); 0 0], 3 x 2"""
    z = p[1] * u[0] * 0
    return [[p[1] * u[0], z], [z, p[1] * u[1]], [z, z]]


def f_scalar(u, p):
    """test/SDE1/sde_scalar_stratonovich.jl:27-47: f = p1 u, one Wiener process for both states"""
    return [p[0] * u[0], p[0] * u[1]]


def G_scalar(u, p):
    return [[p[1] * u[0]], [p[1] * u[1]]]


def G_lv(u, p):
    """sde_lv's diagonal noise (p5 u1, p6 u2) as a 2 x 2 matrix"""
    z = p[4] * u[0] * 0
    return [[p[4] * u[0], z], [z, p[5] * u[1]]]


def G_linear(u, p):
    z = p[1] * u[0] * 0
    return [[p[1] * u[0], z], [z, p[1] * u[1]]]


# name: (f, G, D, P, M); the first six are the plug-ins of examples/sde_noise_families.cuh
FAMILIES = {"sde_roessler": (f_roessler, G_roessler, 2, 4, 2), "sde_mixing": (f_roessler, G_mixing, 2, 4, 2),
            "sde_additive": (f_additive, G_additive, 2, 2, 2), "sde_nonsquare": (f_nonsquare, G_nonsquare, 3, 2, 2),
            "sde_scalar": (f_scalar, G_scalar, 2, 2, 1), "sde_lv_general": (R.f_sde_lv, G_lv, 2, 6, 2),
            "sde_linear_general": (R.f_sde_linear, G_linear, 2, 2, 2)}
PLUGINS = ("sde_roessler", "sde_mixing", "sde_additive", "sde_nonsquare", "sde_scalar", "sde_lv_general")
TWIN = {"sde_lv": "sde_lv_general", "sde_linear": "sde_linear_general"}


def apply(G, u, p, w):
    """G(u, p) w"""
    g = G(u, p)
    return [sum(g[i][j] * w[j] for j in range(len(w))) for i in range(len(g))]


def transformed_drift(f, G, D):
    """f - J_{vec G}' vec G, component k = f_k - sum_ij G_ij dG_ij/du_k (src/sde_tools.jl:29-66)"""
    def F(u, p):
        fv, gv = f(u, p), G(u, p)
        out = []
        for k in range(D):
            gd = G([R.Dual(u[j], 1 if j == k else 0) for j in range(D)], p)
            out.append(fv[k] - sum(gv[i][j] * (gd[i][j].b if isinstance(gd[i][j], R.Dual) else 0)
                                   for i in range(len(gv)) for j in range(len(gv[i]))))
        return out
    return F


# ---- forward and reverse passes ------------------------------------------------------------------------------------

def forward(kind, family, stepper, u0, p, dW, h):
    """EM / EulerHeun from u0 (D arrays) with increments dW[S][M] (kind arrays): -> [u_0, ..., u_S]"""
    f, G, D, _, _ = FAMILIES[family]
    us = [list(u0)]
    u = list(u0)
    for w in dW:
        fv, gw = f(u, p), apply(G, u, p, w)
        ub = [u[j] + h * fv[j] + gw[j] for j in range(D)]
        if stepper == "em":
            u = ub
        else:
            fb, gb = f(ub, p), apply(G, ub, p, w)
            u = [u[j] + h / 2 * (fv[j] + fb[j]) + (gw[j] + gb[j]) / 2 for j in range(D)]
        us.append(u)
    return us


def _terms(kind, F, G, lam, y, p, w):
    """drift (al, am, ay) and diffusion increment (bl, bm, by) of the augmented reverse SDE at (lam, y), increments w"""
    al = [-v for v in R.vjp(kind, F, y, p, lam, "u")]
    am = [-v for v in R.vjp(kind, F, y, p, lam, "p")]
    ay = F(y, p)
    Gw = lambda yy, pp: apply(G, yy, pp, w)
    bl = [-v for v in R.vjp(kind, Gw, y, p, lam, "u")]
    bm = [-v for v in R.vjp(kind, Gw, y, p, lam, "p")]
    by = Gw(y, p)
    return al, am, ay, bl, bm, by


def reverse(kind, family, stepper, sensealg, us, p, dW, h, sos, cost, dgdp=None, ckpt="save", no_start=False):
    """the reverse pass: -> (lam, mu) at t0; arguments as sde_restatement.reverse"""
    f, G, D, P, _ = FAMILIES[family]
    F = transformed_drift(f, G, D) if sensealg == "backsolve" and stepper == "em" else f
    interp = sensealg == "interpolating"
    S = len(dW)
    zero = us[0][0] * 0
    lam, mu, y = [zero] * D, [zero] * P, list(us[S])
    for n in range(S, -1, -1):
        ks = sos.get(n)
        if interp or ckpt == "every" or (ckpt == "save" and ks is not None):
            y = list(us[n])
        if ks is not None and not (interp and no_start and ks == 0):
            dl = cost["dLdu"][ks] if "dLdu" in cost else [cost["a"][j] * y[j] + cost["b"][j] for j in range(D)]
            lam = [lam[j] + dl[j] for j in range(D)]
            if dgdp is not None:
                mu = [mu[q] + dgdp[0][q] * p[q] + dgdp[1][q] for q in range(P)]
        if n == 0:
            break
        w = [-v for v in dW[n - 1]]
        al, am, ay, bl, bm, by = _terms(kind, F, G, lam, y, p, w)
        l1 = [lam[j] - h * al[j] + bl[j] for j in range(D)]
        y1 = [y[j] - h * ay[j] + by[j] for j in range(D)]
        m1 = [mu[q] - h * am[q] + bm[q] for q in range(P)]
        if stepper == "em":
            lam, y, mu = l1, y1, m1
            continue
        if interp:
            y1 = list(us[n - 1])
        al2, am2, ay2, bl2, bm2, by2 = _terms(kind, F, G, l1, y1, p, w)
        lam = [lam[j] - h / 2 * (al[j] + al2[j]) + (bl[j] + bl2[j]) / 2 for j in range(D)]
        y = [y[j] - h / 2 * (ay[j] + ay2[j]) + (by[j] + by2[j]) / 2 for j in range(D)]
        mu = [mu[q] - h / 2 * (am[q] + am2[q]) + (bm[q] + bm2[q]) / 2 for q in range(P)]
    return lam, mu


def gradient(kind_name, family, stepper, sensealg, u0, p, dW, h, saveat, t0=0.0, cost=("affine", 1.0, 0.0), dLdu=None,
             dgdp=None, ckpt="save", no_start=False):
    """one whole gradient, arguments and result as sde_restatement.gradient; dW[S][M][N]"""
    kind = R.Kind(kind_name)
    _, _, D, P, _ = FAMILIES[family]
    u0 = np.asarray(u0, dtype=np.float64)
    N = u0.shape[1]
    p = np.asarray(p, dtype=np.float64)
    if p.ndim == 1:
        p = np.repeat(p[:, None], N, 1)
    with mp.workdps(R.DPS):
        ku0, kp = [kind.arr(x) for x in u0], [kind.arr(x) for x in p]
        kdW = [[kind.arr(x) for x in row] for row in np.asarray(dW, dtype=np.float64)]
        hk = kind.scalar(h)
        us = forward(kind, family, stepper, ku0, kp, kdW, hk)
        vec = lambda x, n: [kind.scalar(v) for v in np.broadcast_to(np.asarray(x, dtype=np.float64), (n,))]
        if cost[0] == "explicit":
            c = {"dLdu": [[kind.arr(x) for x in row] for row in np.asarray(dLdu, dtype=np.float64)]}
        else:
            c = {"a": vec(cost[1], D), "b": vec(cost[2], D)}
        dg = None if dgdp is None else (vec(dgdp[0], P), vec(dgdp[1], P))
        lam, mu = reverse(kind, family, stepper, sensealg, us, kp, kdW, hk, R.save_table(saveat, t0, h), c, dg, ckpt, no_start)
        return (np.array([kind.f64(v) for v in lam]), np.array([kind.f64(v) for v in mu]),
                np.array([[kind.f64(v) for v in u] for u in us]))


def loss(family, stepper, u0, p, dW, h, saveat, a=1.0, b=0.0, t0=0.0):
    """sum over the save times of sum_j a/2 u_j^2 + b u_j along the long-double forward solve: -> [N]"""
    kind = R.Kind("ld")
    us = forward(kind, family, stepper, [kind.arr(x) for x in np.asarray(u0, dtype=np.float64)],
                 [kind.arr(x) for x in np.asarray(p, dtype=np.float64)],
                 [[kind.arr(x) for x in row] for row in np.asarray(dW, dtype=np.float64)], R.LD(h))
    out = 0
    for n in R.save_table(saveat, t0, h):
        out = out + sum(R.LD(a) / 2 * v * v + R.LD(b) * v for v in us[n])
    return out


# ---- closed forms along one path (Stratonovich solutions), cost sum_k sum_j a/2 u_j(t_k)^2 + b u_j(t_k) ----------------

def closed_gradient(family, u0, p, W, ts, a=1.0, b=0.0):
    """(du0[D], dp[P]) of one member: W[K][M] the Brownian path at the save times ts, u0 [D], p [P]"""
    from scipy.linalg import expm_frechet
    u0, p = np.asarray(u0, dtype=np.float64), np.asarray(p, dtype=np.float64)
    D, P = FAMILIES[family][2], FAMILIES[family][3]
    du0, dp = np.zeros(D), np.zeros(P)
    for t, w in zip(ts, W):
        if family == "sde_roessler":
            swap = np.array([[0.0, 1.0], [1.0, 0.0]])
            X = (p[0] * np.eye(2) + p[1] * swap) * t + (p[2] * np.eye(2) + p[3] * swap) * (w[0] + w[1])
            dX = [t * np.eye(2), t * swap, (w[0] + w[1]) * np.eye(2), (w[0] + w[1]) * swap]
            E = expm_frechet(X, dX[0], compute_expm=True)[0]
            u = E @ u0
            dl = a * u + b
            du0 += E.T @ dl
            for q in range(4):
                dp[q] += dl @ (expm_frechet(X, dX[q], compute_expm=False) @ u0)
            continue
        if family == "sde_scalar":
            ex = np.exp(p[0] * t + p[1] * w[0]) * np.ones(2)
            dex = [t * ex, w[0] * ex]
        elif family == "sde_nonsquare":
            ex = np.exp(p[0] * t + p[1] * np.array([w[0], w[1], 0.0]))
            dex = [t * ex, np.array([w[0], w[1], 0.0]) * ex]
        else:
            raise KeyError(family)
        u = u0 * ex
        dl = a * u + b
        du0 += dl * ex
        for q in range(2):
            dp[q] += dl @ (u0 * dex[q])
    return du0, dp


# ---- the configuration matrix of tests/test_gpu_sde_noise.py ----------------------------------------------------------

P_NOMINAL = {"sde_roessler": [-1.5, 0.05, 0.2, 0.01], "sde_mixing": [-1.5, 0.05, 0.2, 0.01], "sde_additive": [1.0, 0.3],
             "sde_nonsquare": [1.0, 0.1], "sde_scalar": [1.01, 0.87], "sde_lv_general": [1.5, 1.0, 3.0, 1.0, 0.1, 0.1]}
U0_NOMINAL = {"sde_roessler": [0.75, 0.5], "sde_mixing": [0.75, 0.5], "sde_additive": [0.2, -0.1], "sde_nonsquare": [1.0, 0.8, 0.6],
              "sde_scalar": [0.6, 0.3], "sde_lv_general": [1.0, 1.0]}
FACTORS = (("family", PLUGINS), ("stepper", ("em", "euler_heun")), ("sa", tuple(R.SENSEALGS)),
           ("cost", ("scalar", "vector_dgdp", "explicit")), ("p", ("shared", "member")), ("noise", ("regen", "stored", "dW")),
           ("saveat", tuple(R.SAVEATS)))


def allowed(c):
    """EM + BacksolveAdjoint is refused for general noise; no_start as in sde_restatement"""
    return R._allowed(c) and not (c["stepper"] == "em" and c["sa"].startswith("bs"))


def config_matrix():
    """every pair of factor levels and every reverse-kernel instantiation of every family at least once: greedy, deterministic"""
    names = [n for n, _ in FACTORS]
    allc = [dict(zip(names, v)) for v in itertools.product(*[lv for _, lv in FACTORS])]
    allc = [c for c in allc if allowed(c)]

    def items(c):
        out = {("pair", a, c[a], b, c[b]) for a, b in itertools.combinations(names, 2)}
        out.add(("kernel",) + R._kernel_of(c))
        return out
    need = set().union(*(items(c) for c in allc))
    chosen = []
    while need:
        best = max(allc, key=lambda c: len(items(c) & need))
        chosen.append(best)
        need -= items(best)
    return chosen


def costs(D):
    return {"scalar": (1.0, -0.25), "vector_dgdp": (np.linspace(1.0, 0.5, D), np.linspace(-0.3, 0.2, D))}


def problem(c, N, seed):
    """the inputs of a configuration: u0[D][N], p ([P] or [P][N]), cost tuple, dgdp or None, dLdu or None"""
    rng = np.random.default_rng(seed)
    fam = c["family"]
    _, _, D, P, _ = FAMILIES[fam]
    u0 = np.asarray(U0_NOMINAL[fam])[:, None] * np.exp(0.05 * rng.standard_normal((D, N)))
    p = np.asarray(P_NOMINAL[fam], dtype=np.float64)
    if c["p"] == "member":
        p = p[:, None] * np.exp(0.02 * rng.standard_normal((P, N)))
    K = len(R.SAVEATS[c["saveat"]])
    dLdu = rng.uniform(0.5, 1.5, (K, D, N)) if c["cost"] == "explicit" else None
    cost = ("explicit",) if c["cost"] == "explicit" else ("affine",) + costs(D)[c["cost"]]
    dgdp = (np.linspace(0.2, 0.7, P), np.linspace(-0.1, 0.15, P)) if c["cost"] == "vector_dgdp" else None
    return u0, p, cost, dgdp, dLdu
