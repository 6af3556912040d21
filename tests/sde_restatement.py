"""The diagonal-noise SDE path (csrc/sde_em.cuh) restated in plain Python, generic over the number type: mpmath at 40
digits, np.longdouble, or float64, vectorised over the ensemble members.  The only model inputs are the right-hand sides
of the reference's SDE test problems (f and g below); every derivative comes from complex steps of those (the Ito
correction's inner Jacobian from a dual number), never from families.cuh or oracle/adjoint_oracle.c.

* The noise: Philox4x32-10 (Salmon et al. 2011) in integer arithmetic with key = (seed lo, seed hi) and counter =
  (member lo, member hi, step, pair); two 53-bit uniforms ((r0 << 21) ^ (r1 >> 11) + 0.5) 2^-53 formed in float64 as
  the device forms them (the + 0.5 rounds to even above 2^52); Box-Muller z0 = rad cospi(2 u2), z1 = rad sinpi(2 u2),
  rad = sqrt(-2 log u1); component 2q takes z0 of pair q and component 2q + 1 its z1; dW = sqrt(h) z.
* The forward pass: Euler-Maruyama and EulerHeun on the dt grid.
* The reverse pass of SDEAdjointProblem, stepping dt = -h with the increment -dW_{n-1}:
  BacksolveAdjoint z = [lam; mu; y] (src/backsolve_adjoint.jl:274-419), its drift the Ito-transformed f - (dg/du)' g
  (StochasticTransformedFunction, src/sde_tools.jl, full factor) for the Ito solver EM only (:327-345);
  InterpolatingAdjoint z = [lam; mu] with y read from the forward solution (src/interpolating_adjoint.jl:453-613);
  the diagonal-noise diffusion VJPs of src/derivative_wrappers.jl:1165-1211.  At every grid point, in this order: the
  checkpoint reset of y (at every save time, at every step, or never; always for Interpolating), then the loss jump
  (src/adjoint_common.jl:754-821) evaluated at the current y, with its dgdp part; no_start skips the first save time
  for every sensealg but Backsolve.
* Near-miss variants of the algorithm, used to show that the tests' tolerances separate the device from them.
"""

import numpy as np

import mpmath as mp

LD = np.longdouble
DPS = 40
MASK32 = np.uint64(0xFFFFFFFF)
PHILOX_M = (np.uint64(0xD2511F53), np.uint64(0xCD9E8D57))
PHILOX_W = (np.uint64(0x9E3779B9), np.uint64(0xBB67AE85))
TWO_M53 = 2.0 ** -53
LD_PI = LD("3.14159265358979323846264338327950288")
VARIANTS = ("half_ito", "plus_dw", "dw_of_step_n", "eh_corrector_at_yn", "reset_after_jump")


# ---- the noise -----------------------------------------------------------------------------------------------------

def philox4x32_10(ctr, key):
    """Philox4x32-10 on counter words (c0, c1, c2, c3) and key words (k0, k1), ints or arrays: -> 4 uint64 arrays of
    32-bit words"""
    c = [np.asarray(x, dtype=np.uint64) & MASK32 for x in ctr]
    k = [np.asarray(x, dtype=np.uint64) & MASK32 for x in key]
    for _ in range(10):
        p0, p1 = PHILOX_M[0] * c[0], PHILOX_M[1] * c[2]       # 32 x 32 -> 64 bits: exact in uint64
        hi0, lo0, hi1, lo1 = p0 >> np.uint64(32), p0 & MASK32, p1 >> np.uint64(32), p1 & MASK32
        c = [hi1 ^ c[1] ^ k[0], lo1, hi0 ^ c[3] ^ k[1], lo0]
        k = [(k[0] + PHILOX_W[0]) & MASK32, (k[1] + PHILOX_W[1]) & MASK32]
    return c


def words(seed, member, step, pair):
    """the generator's four words for (seed, member, step, pair); member may be an array (uint64)"""
    seed, member = np.uint64(seed), np.asarray(member, dtype=np.uint64)
    return philox4x32_10((member & MASK32, member >> np.uint64(32), step, pair), (seed & MASK32, seed >> np.uint64(32)))


def uniforms(r):
    """the two float64 uniforms in (0, 1) of one Philox output, formed exactly as the device forms them"""
    a = (r[0] << np.uint64(21)) ^ (r[1] >> np.uint64(11))
    b = (r[2] << np.uint64(21)) ^ (r[3] >> np.uint64(11))
    return (a.astype(np.float64) + 0.5) * TWO_M53, (b.astype(np.float64) + 0.5) * TWO_M53


def box_muller(u1, u2, kind):
    """(z0, z1, rad) of float64 uniforms, in long double ('ld') or 40 digits ('mp', object arrays)"""
    if kind == "ld":
        rad = np.sqrt(-2 * np.log(u1.astype(LD)))
        ang = 2 * LD_PI * u2.astype(LD)
        return rad * np.cos(ang), rad * np.sin(ang), rad
    with mp.workdps(DPS):
        rad = np.array([mp.sqrt(-2 * mp.log(mp.mpf(float(v)))) for v in u1], dtype=object)
        c = np.array([mp.cospi(2 * mp.mpf(float(v))) for v in u2], dtype=object)
        s = np.array([mp.sinpi(2 * mp.mpf(float(v))) for v in u2], dtype=object)
        return rad * c, rad * s, rad


def normal_pair(seed, member, step, pair, kind="ld"):
    return box_muller(*uniforms(words(seed, member, step, pair)), kind)


def increments(seed, traj_offset, N, S, m, h, kind="ld"):
    """-> (dW[S][m][N], rad[S][m][N]) of members traj_offset .. traj_offset + N - 1, in long double or 40 digits"""
    member = np.uint64(traj_offset) + np.arange(N, dtype=np.uint64)
    dt = LD if kind == "ld" else object
    dW, rad = np.zeros((S, m, N), dtype=dt), np.zeros((S, m, N), dtype=dt)
    with mp.workdps(DPS):
        sq = np.sqrt(LD(h)) if kind == "ld" else mp.sqrt(mp.mpf(h))
        for n in range(S):
            for q in range((m + 1) // 2):
                z0, z1, r = normal_pair(seed, member, n, q, kind)
                dW[n, 2 * q], rad[n, 2 * q] = sq * z0, r
                if 2 * q + 1 < m:
                    dW[n, 2 * q + 1], rad[n, 2 * q + 1] = sq * z1, r
    return dW, rad


# ---- the test problems ---------------------------------------------------------------------------------------------

def f_sde_lv(u, p):
    """Lotka-Volterra drift of test/Core1/concrete_solve_derivatives.jl:736-760"""
    return [p[0] * u[0] - p[1] * u[0] * u[1], -p[2] * u[1] + p[3] * u[0] * u[1]]


def g_sde_lv(u, p):
    """its diagonal noise sigma(u, p) = (p[5] u[1], p[6] u[2]) (1-based there)"""
    return [p[4] * u[0], p[5] * u[1]]


def f_sde_linear(u, p):
    """the linear SDE of test/SDE1/sde_stratonovich.jl:22-35, two components: f = p[1] u, sigma = p[2] u"""
    return [p[0] * u[0], p[0] * u[1]]


def g_sde_linear(u, p):
    return [p[1] * u[0], p[1] * u[1]]


FAMILIES = {"sde_lv": (f_sde_lv, g_sde_lv, 2, 6), "sde_linear": (f_sde_linear, g_sde_linear, 2, 2)}


class Dual:
    """a + b eps with eps^2 = 0 over any number type (arrays included): the Ito correction's inner derivative"""
    __array_ufunc__ = None          # numpy arrays defer to the reflected operators below

    def __init__(self, a, b):
        self.a, self.b = a, b

    def __add__(self, o):
        return Dual(self.a + o.a, self.b + o.b) if isinstance(o, Dual) else Dual(self.a + o, self.b)
    __radd__ = __add__

    def __sub__(self, o):
        return Dual(self.a - o.a, self.b - o.b) if isinstance(o, Dual) else Dual(self.a - o, self.b)

    def __rsub__(self, o):
        return Dual(o - self.a, -self.b)

    def __neg__(self):
        return Dual(-self.a, -self.b)

    def __mul__(self, o):
        return Dual(self.a * o.a, self.a * o.b + self.b * o.a) if isinstance(o, Dual) else Dual(self.a * o, self.b * o)
    __rmul__ = __mul__


def ito_drift(f, g, D, factor=1):
    """f - factor (dg/du)' g: StochasticTransformedFunction of src/sde_tools.jl (factor 1; factor 1/2 is a near miss)"""
    def F(u, p):
        gv, fv = g(u, p), f(u, p)
        out = []
        for c in range(D):
            gd = g([Dual(u[j], 1 if j == c else 0) for j in range(D)], p)
            out.append(fv[c] - factor * sum(gv[i] * (gd[i].b if isinstance(gd[i], Dual) else 0) for i in range(D)))
        return out
    return F


# ---- number kinds --------------------------------------------------------------------------------------------------

class Kind:
    """'mp' (object arrays of mpf, 40 digits), 'ld' (np.longdouble) or 'f64' (float64)"""

    def __init__(self, name):
        self.name = name
        if name == "mp":
            self.d = mp.mpf("1e-30")
            self.idelta = mp.mpc(0, self.d)
        elif name == "ld":
            self.d = LD("1e-30")
            self.idelta = np.clongdouble(1j) * self.d
        else:
            self.d = 1e-30
            self.idelta = 1e-30j

    def scalar(self, x):
        """a float64 value, exactly"""
        return mp.mpf(float(x)) if self.name == "mp" else (LD(float(x)) if self.name == "ld" else float(x))

    def arr(self, a):
        a = np.asarray(a, dtype=np.float64)
        if self.name == "mp":
            return np.array([mp.mpf(float(v)) for v in a.ravel()], dtype=object).reshape(a.shape)
        return a.astype(LD) if self.name == "ld" else a.copy()

    def cplx(self, a):
        if self.name == "mp":
            return np.array([mp.mpc(v) for v in a], dtype=object)
        return np.asarray(a).astype(np.clongdouble if self.name == "ld" else np.complex128)

    def imag(self, z):
        return np.array([mp.im(v) for v in z], dtype=object) if self.name == "mp" else np.asarray(z).imag

    def f64(self, a):
        return np.array([float(v) for v in np.ravel(a)]).reshape(np.shape(a)) if self.name == "mp" else np.asarray(a, dtype=np.float64)


def vjp(kind, F, y, p, l, wrt):
    """(dF/du)' l or (dF/dp)' l by complex steps of l' F(y, p); y, p, l lists of member arrays"""
    yc, pc = [kind.cplx(v) for v in y], [kind.cplx(v) for v in p]
    out = []
    for c in range(len(y) if wrt == "u" else len(p)):
        yy, pp = list(yc), list(pc)
        if wrt == "u":
            yy[c] = yy[c] + kind.idelta
        else:
            pp[c] = pp[c] + kind.idelta
        out.append(kind.imag(sum(l[r] * v for r, v in enumerate(F(yy, pp)))) / kind.d)
    return out


def g_diag_du(kind, g, y, p):
    """dg_i/du_i, the diagonal-noise Jacobian (src/derivative_wrappers.jl:1197-1199)"""
    yc, pc = [kind.cplx(v) for v in y], [kind.cplx(v) for v in p]
    out = []
    for i in range(len(y)):
        yy = list(yc)
        yy[i] = yy[i] + kind.idelta
        out.append(kind.imag(g(yy, pc)[i]) / kind.d)
    return out


# ---- forward and reverse passes ------------------------------------------------------------------------------------

def forward(kind, family, stepper, u0, p, dW, h):
    """EM / EulerHeun from u0 (D arrays) with increments dW[S][m] (kind arrays): -> [u_0, ..., u_S]"""
    f, g, D, _ = FAMILIES[family]
    us = [list(u0)]
    u = list(u0)
    for w in dW:
        fv, gv = f(u, p), g(u, p)
        ub = [u[j] + h * fv[j] + gv[j] * w[j] for j in range(D)]
        if stepper == "em":
            u = ub
        else:
            fb, gb = f(ub, p), g(ub, p)
            u = [u[j] + h / 2 * (fv[j] + fb[j]) + (gv[j] + gb[j]) / 2 * w[j] for j in range(D)]
        us.append(u)
    return us


def _terms(kind, F, g, lam, y, p, w):
    """drift (al, am, ay) and diffusion increment (bl, bm, by) of the augmented reverse SDE at (lam, y), increments w"""
    al = [-v for v in vjp(kind, F, y, p, lam, "u")]
    am = [-v for v in vjp(kind, F, y, p, lam, "p")]
    ay = F(y, p)
    gd = g_diag_du(kind, g, y, p)
    bl = [-gd[j] * lam[j] * w[j] for j in range(len(y))]
    bm = [-v for v in vjp(kind, g, y, p, [lam[j] * w[j] for j in range(len(y))], "p")]
    by = [gv * wj for gv, wj in zip(g(y, p), w)]
    return al, am, ay, bl, bm, by


def reverse(kind, family, stepper, sensealg, us, p, dW, h, sos, cost, dgdp=None, ckpt="save", no_start=False, variant=None):
    """the reverse pass: -> (lam, mu) at t0.  sos: {grid index: save index}; cost: dict(a=[D], b=[D]) (affine,
    dg/du = a u + b at the current y) or dict(dLdu=[K][D] member arrays) (explicit); dgdp: (c[P], e[P]) of the
    parameter part c p + e or None; ckpt: 'save' | 'every' | 'never' (Backsolve); variant: None or one of VARIANTS"""
    f, g, D, P = FAMILIES[family]
    ito = sensealg == "backsolve" and stepper == "em"
    F = ito_drift(f, g, D, 0.5 if variant == "half_ito" else 1) if ito else f
    interp = sensealg == "interpolating"
    S = len(dW)
    zero = us[0][0] * 0
    st = {"lam": [zero] * D, "mu": [zero] * P, "y": list(us[S])}

    def reset(n, ks):
        if interp or ckpt == "every" or (ckpt == "save" and ks is not None):
            st["y"] = list(us[n])

    def jump(ks):
        if ks is None or (interp and no_start and ks == 0):
            return
        y = st["y"]
        dl = cost["dLdu"][ks] if "dLdu" in cost else [cost["a"][j] * y[j] + cost["b"][j] for j in range(D)]
        st["lam"] = [st["lam"][j] + dl[j] for j in range(D)]
        if dgdp is not None:
            st["mu"] = [st["mu"][q] + dgdp[0][q] * p[q] + dgdp[1][q] for q in range(P)]

    for n in range(S, -1, -1):
        ks = sos.get(n)
        if variant == "reset_after_jump":
            jump(ks)
            reset(n, ks)
        else:
            reset(n, ks)
            jump(ks)
        lam, mu, y = st["lam"], st["mu"], st["y"]
        if n == 0:
            break
        wn = dW[n % S] if variant == "dw_of_step_n" else dW[n - 1]
        w = list(wn) if variant == "plus_dw" else [-v for v in wn]
        al, am, ay, bl, bm, by = _terms(kind, F, g, lam, y, p, w)
        l1 = [lam[j] - h * al[j] + bl[j] for j in range(D)]
        y1 = [y[j] - h * ay[j] + by[j] for j in range(D)]
        m1 = [mu[q] - h * am[q] + bm[q] for q in range(P)]
        if stepper == "em":
            st.update(lam=l1, y=y1, mu=m1)
            continue
        if interp:
            y1 = list(us[n] if variant == "eh_corrector_at_yn" else us[n - 1])
        al2, am2, ay2, bl2, bm2, by2 = _terms(kind, F, g, l1, y1, p, w)
        st.update(lam=[lam[j] - h / 2 * (al[j] + al2[j]) + (bl[j] + bl2[j]) / 2 for j in range(D)],
                  y=[y[j] - h / 2 * (ay[j] + ay2[j]) + (by[j] + by2[j]) / 2 for j in range(D)],
                  mu=[mu[q] - h / 2 * (am[q] + am2[q]) + (bm[q] + bm2[q]) / 2 for q in range(P)])
    return st["lam"], st["mu"]


def save_table(saveat, t0, h):
    """{grid index n: save index k} of save times on the dt grid"""
    return {int(round((t - t0) / h)): k for k, t in enumerate(saveat)}


def gradient(kind_name, family, stepper, sensealg, u0, p, dW, h, saveat, t0=0.0, cost=("affine", 1.0, 0.0), dLdu=None,
             dgdp=None, ckpt="save", no_start=False, variant=None):
    """one whole gradient in the given number kind from float64 inputs (taken exactly): u0[D][M], p[P] or [P][M],
    dW[S][m][M], cost ("affine", a, b) with scalar or per-component a, b, or ("explicit",) with dLdu[K][D][M];
    dgdp (c[P], e[P]) or None.  -> (du0[D][M], dp[P][M] per member, u[S+1][D][M]) in float64"""
    kind = Kind(kind_name)
    _, _, D, P = FAMILIES[family]
    u0 = np.asarray(u0, dtype=np.float64)
    M = u0.shape[1]
    p = np.asarray(p, dtype=np.float64)
    if p.ndim == 1:
        p = np.repeat(p[:, None], M, 1)
    with mp.workdps(DPS):
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
        lam, mu = reverse(kind, family, stepper, sensealg, us, kp, kdW, hk, save_table(saveat, t0, h), c, dg, ckpt, no_start, variant)
        return (np.array([kind.f64(v) for v in lam]), np.array([kind.f64(v) for v in mu]),
                np.array([[kind.f64(v) for v in u] for u in us]))


# ---- the configuration matrix of tests/test_sde_restatement.py and tests/test_gpu_sde_reference.py -------------------

T_END, H, S_STEPS = 1.0, 0.025, 40
GRID = np.linspace(0.0, T_END, S_STEPS + 1)
SAVEATS = {"full": GRID, "no_t0": GRID[[3, 10, 17, 29, 40]], "no_T": GRID[[0, 6, 13, 22, 31]], "single": GRID[[21]]}
SENSEALGS = {"bs_save": ("backsolve", "save", False), "bs_every": ("backsolve", "every", False), "bs_never": ("backsolve", "never", False),
             "interp": ("interpolating", "save", False), "interp_no_start": ("interpolating", "save", True)}
FACTORS = (("family", ("sde_lv", "sde_linear")), ("stepper", ("em", "euler_heun")), ("sa", tuple(SENSEALGS)),
           ("cost", ("scalar", "vector_dgdp", "explicit")), ("p", ("shared", "member")), ("noise", ("regen", "stored", "dW")),
           ("saveat", tuple(SAVEATS)))
P_NOMINAL = {"sde_lv": [1.5, 1.0, 3.0, 1.0, 0.1, 0.1], "sde_linear": [1.01, 0.87]}
U0_NOMINAL = {"sde_lv": [1.0, 1.0], "sde_linear": [1.0, 0.5]}
COSTS = {"scalar": (1.0, -0.25), "vector_dgdp": ([1.0, 0.5], [-0.3, 0.2])}


def _allowed(c):
    # no_start marks a forward solve that saved t0 without using it (src/concrete_solve.jl: no_start = !save_start && t0 in ts)
    return not (c["sa"] == "interp_no_start" and c["saveat"] in ("no_t0", "single"))


def _kernel_of(c):
    """the sde_backsolve_kernel instantiation a configuration launches (family, EulerHeun, shared p, explicit cost, interp)"""
    return (c["family"], c["stepper"], c["p"], c["cost"] == "explicit", c["sa"].startswith("interp"))


def config_matrix():
    """every pair of factor levels and every reverse-kernel instantiation at least once: greedy, deterministic"""
    import itertools
    names = [n for n, _ in FACTORS]
    allc = [dict(zip(names, v)) for v in itertools.product(*[lv for _, lv in FACTORS])]
    allc = [c for c in allc if _allowed(c)]

    def items(c):
        out = {("pair", a, c[a], b, c[b]) for a, b in itertools.combinations(names, 2)}
        out.add(("kernel",) + _kernel_of(c))
        return out
    need = set().union(*(items(c) for c in allc))
    chosen = []
    while need:
        best = max(allc, key=lambda c: len(items(c) & need))
        chosen.append(best)
        need -= items(best)
    return chosen


def problem(c, N, seed):
    """the inputs of a configuration: u0[2][N], p ([P] or [P][N]), cost tuple, dgdp or None, dLdu or None"""
    rng = np.random.default_rng(seed)
    fam = c["family"]
    P = FAMILIES[fam][3]
    u0 = np.asarray(U0_NOMINAL[fam])[:, None] * np.exp(0.05 * rng.standard_normal((2, N)))
    p = np.asarray(P_NOMINAL[fam], dtype=np.float64)
    if c["p"] == "member":
        p = p[:, None] * np.exp(0.02 * rng.standard_normal((P, N)))
    K = len(SAVEATS[c["saveat"]])
    dLdu = rng.uniform(0.5, 1.5, (K, 2, N)) if c["cost"] == "explicit" else None
    cost = ("explicit",) if c["cost"] == "explicit" else ("affine",) + COSTS[c["cost"]]
    dgdp = (np.linspace(0.2, 0.7, P), np.linspace(-0.1, 0.15, P)) if c["cost"] == "vector_dgdp" else None
    return u0, p, cost, dgdp, dLdu


def label(c):
    return "-".join(str(c[n]) for n, _ in FACTORS)


def rel_err(x, ref, part=None):
    """|x - ref| per component over max(|ref|, 1e-6 of the member's largest |ref|); arrays [C][M] or [C].  part: a
    known summand of ref (the dgdp part of dp); the scale is then at least the larger of the two summands, so that a
    component in which they cancel is judged by the rounding of its terms"""
    x, ref = np.asarray(x, dtype=np.float64), np.asarray(ref, dtype=np.float64)
    if ref.ndim == 1:
        x, ref = x[:, None], ref[:, None]
    scale = np.maximum(np.abs(ref), 1e-6 * np.abs(ref).max(axis=0, keepdims=True))
    if part is not None:
        part = np.broadcast_to(np.asarray(part, dtype=np.float64).reshape(ref.shape[0], -1), ref.shape)
        scale = np.maximum(scale, np.maximum(np.abs(part), np.abs(ref - part)))
    return np.abs(x - ref) / np.where(scale > 0, scale, 1.0)
