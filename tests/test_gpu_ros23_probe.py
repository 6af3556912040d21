"""The device functions behind the Rosenbrock23 kernels (csrc/ros23.cuh, csrc/families.cuh), one at a time, through
tests/csrc/ros23_probe.cu: the production functions wrapped in small kernels, no copies.

* Family derivatives (LV, Lorenz, Robertson, BouncingBall, Relax and the LvClone plug-in example): `jac`, `djac`, `dvjp_p`,
  `vjp_u`, `vjp_p` against complex-step differentiation of a numpy restatement of `f` alone.  First derivatives take one
  complex step; the second derivatives `djac(p, yd) = d/de J(u + e yd)` and `dvjp_p(u, yd, l) = d/de (df/dp)'l at u + e yd`
  take two independent imaginary units (bicomplex numbers), so no derivative is formed by a difference quotient.  Bound:
  1e-14 relative per entry, the scale taken from the matrix (Jacobians) or the row max of |l|'|J| (the vector-Jacobian
  products).
* `lu_factor` / `lu_solve` (D = 1, 2, 3): exact on dyadic systems, the pivot row pinned (zero leading pivot, ties between
  equal magnitudes keep the first row), `false` on singular matrices, and Robertson's W = I - h d J (forward, h > 0) and
  I + h d J' (the lambda block of the reverse solves, h < 0) for |h| in [1e-4, 90] against a 40-digit solve within
  4 D cond(W) eps.  These found lu_factor swapping whole rows, multipliers included, while lu_solve replays the swaps one
  column at a time: for D = 3 a pivot off the diagonal in column c >= 1 paired the multipliers with the wrong rows (75 of
  the 200 dyadic systems).  Whether a solve meets such a pivot depends on W; none of the Rosenbrock23 runs of the suite is
  known to have, and a W-method still converges with a wrong W.
* `FwdDense<D>::eval` on synthetic forward records: the interval chosen, y bitwise (the restatement evaluates the same
  operations, with the fused multiply-adds the compiler emits for it), yd against a complex-step derivative to 1e-14.
* `step_factor_I` and `tstop_snap` bitwise on their edges.

Observed on an H100 SXM (700 W): cond(W) up to 3.6e5 (forward) and 4.0e5 (reverse), err / (cond(W) eps) at most 0.61 and
0.55.  With tests/test_gpu_ros23_reference.py, test_gpu_parity_ros23.py and test_gpu_family_plugin.py the Rosenbrock23 tests
took 66 s there, the probe's compilation ~2 s of it.
"""
import ctypes as C
import os
import subprocess
from fractions import Fraction

import numpy as np
import pytest

from scimlsensitivity_jl_b200 import _lib
from ros23_restatement import dense_interval, f_ball, f_lorenz, f_lv, f_relax, f_robertson, fma

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
CSRC = os.path.join(ROOT, "scimlsensitivity.jl_b200", "csrc")
PROBE = os.path.join(ROOT, "tests", "csrc", "ros23_probe.cu")

ROS_D = 0.29289321881345247559915563789515
IC = 1.0 - 2 * ROS_D                     # (1 - 2d) as the kernels fold it
EPS100 = 100 * 2.220446049250313e-16


@pytest.fixture(scope="session")
def ros23_probe_so(tmp_path_factory):
    """ros23_probe.cu built with the library's nvcc flags, once per session, outside the source tree."""
    so = str(tmp_path_factory.mktemp("ros23_probe") / "libros23_probe.so")
    cmd = [_lib.nvcc_path(), "-gencode", "arch=compute_90a,code=sm_90a", "-O3", "-std=c++17", "-I", CSRC,
           "-Xcompiler", "-fPIC", "-shared", PROBE, "-o", so]
    res = subprocess.run(cmd, capture_output=True, text=True)
    assert res.returncode == 0, res.stdout[-3000:] + res.stderr[-3000:]
    return so


def test_ros23_probe_compiles_for_sm90a(ros23_probe_so):
    """No GPU needed: a header change that breaks the probes fails here."""
    lib = C.CDLL(ros23_probe_so)
    for name in ("probe_family", "probe_lu", "probe_dense", "probe_scalars"):
        getattr(lib, name)


@pytest.fixture(scope="module")
def probe(ros23_probe_so):
    lib = C.CDLL(ros23_probe_so)
    vp, i = C.c_void_p, C.c_int
    lib.probe_family.argtypes = [i, i, vp, vp, vp, vp, vp]
    lib.probe_lu.argtypes = [i, i, vp, vp, vp, vp, vp, vp]
    lib.probe_dense.argtypes = [i, vp, vp, vp, vp, C.c_longlong, i, vp, vp, vp, vp, vp]
    lib.probe_scalars.argtypes = [i, vp, vp, vp, vp, vp]
    return lib


def _dev(x, dtype=None):
    import torch
    x = np.ascontiguousarray(x)
    if dtype is None:
        dtype = torch.float64 if x.dtype.kind == "f" else torch.int32
    return torch.tensor(x, dtype=dtype, device="cuda")


def _zeros(shape, dtype="f"):
    import torch
    return torch.zeros(shape, dtype=torch.float64 if dtype == "f" else torch.int32, device="cuda")


def _check(rc):
    assert rc == 0, f"probe launch failed: cudaError {rc}"


# ------------------------------------------------------------------------------------------------------------------------
# family derivatives: f restated, everything else by complex steps


class BC:
    """bicomplex number a + b j (a, b complex, i j = j i, j^2 = -1): two independent complex steps, enough for the
    polynomial right-hand sides (+, -, * only)"""

    def __init__(self, a, b=0j):
        self.a, self.b = complex(a), complex(b)

    @staticmethod
    def _c(x):
        return x if isinstance(x, BC) else BC(x)

    def __add__(self, o):
        o = BC._c(o)
        return BC(self.a + o.a, self.b + o.b)

    __radd__ = __add__

    def __sub__(self, o):
        o = BC._c(o)
        return BC(self.a - o.a, self.b - o.b)

    def __rsub__(self, o):
        return BC._c(o) - self

    def __neg__(self):
        return BC(-self.a, -self.b)

    def __mul__(self, o):
        o = BC._c(o)
        return BC(self.a * o.a - self.b * o.b, self.a * o.b + self.b * o.a)

    __rmul__ = __mul__


# probe index, f, D, P
FAMILIES = {"lv": (0, f_lv, 2, 4), "lorenz": (1, f_lorenz, 3, 3), "robertson": (2, f_robertson, 3, 3), "ball": (3, f_ball, 2, 2),
            "relax": (4, f_relax, 1, 2), "lv_clone": (5, f_lv, 2, 4)}
DELTA = 1e-60


def cs_first(f, u, p, D, P):
    """J[r][c] = df_r/du_c, F[r][q] = df_r/dp_q (one complex step each)"""
    J, F = np.zeros((D, D)), np.zeros((D, P))
    for c in range(D):
        uc = [complex(x) for x in u]
        uc[c] += 1j * DELTA
        J[:, c] = [v.imag / DELTA for v in map(complex, f(uc, [complex(x) for x in p]))]
    for q in range(P):
        pc = [complex(x) for x in p]
        pc[q] += 1j * DELTA
        F[:, q] = [complex(v).imag / DELTA for v in f([complex(x) for x in u], pc)]
    return J, F


def cs_second(f, u, p, ud, D, P):
    """dJ[r][c] = d/de df_r/du_c (u + e ud), dF[r][q] = d/de df_r/dp_q (u + e ud): i-step on u_c / p_q, j-step along ud"""
    dJ, dF = np.zeros((D, D)), np.zeros((D, P))
    for c in range(D):
        uc = [BC(u[k] + (1j * DELTA if k == c else 0.0), DELTA * ud[k]) for k in range(D)]
        dJ[:, c] = [v.b.imag / DELTA ** 2 for v in map(BC._c, f(uc, [BC(x) for x in p]))]
    for q in range(P):
        uc = [BC(u[k], DELTA * ud[k]) for k in range(D)]
        pc = [BC(p[k] + (1j * DELTA if k == q else 0.0)) for k in range(P)]
        dF[:, q] = [v.b.imag / DELTA ** 2 for v in map(BC._c, f(uc, pc))]
    return dJ, dF


def _points(name, n, rng):
    """-> u[n][D], p[n][P], ud[n][D], l[n][D] at the magnitudes the solves meet"""
    _, f, D, P = FAMILIES[name]
    if name in ("lv", "lv_clone"):
        u = np.exp(0.5 * rng.standard_normal((n, 2)))
        p = np.array([1.5, 1.0, 3.0, 1.0]) * np.exp(0.1 * rng.standard_normal((n, 4)))
    elif name == "lorenz":
        u = 10.0 * rng.standard_normal((n, 3))
        p = np.array([10.0, 28.0, 8.0 / 3.0]) * np.exp(0.05 * rng.standard_normal((n, 3)))
    elif name == "robertson":      # the real magnitudes: k = (0.04, 3e7, 1e4), y2 ~ 1e-5 .. 4e-5, ydot from the flow
        y0 = rng.uniform(0.3, 1.0, n)
        y1 = rng.uniform(1e-5, 4e-5, n)
        u = np.stack([y0, y1, 1.0 - y0 - y1], axis=1)
        p = np.array([0.04, 3e7, 1e4]) * np.exp(0.05 * rng.standard_normal((n, 3)))
    elif name == "ball":
        u = rng.standard_normal((n, 2)) * [5.0, 10.0]
        p = np.stack([rng.uniform(1, 20, n), rng.uniform(0.5, 1, n)], axis=1)
    else:
        u = rng.standard_normal((n, 1))
        p = rng.standard_normal((n, 2))
    if name == "robertson":
        ud = np.array([f(list(u[i]), list(p[i])) for i in range(n)])
    else:
        ud = rng.standard_normal((n, D))
    l = rng.standard_normal((n, D)) * (10.0 ** rng.uniform(-2, 2, (n, 1)))
    return u, p, ud, l


def _rel_err(a, ref, scale):
    scale = np.maximum(scale, 1e-300)
    return np.abs(a - ref) / scale


@pytest.mark.gpu
@pytest.mark.parametrize("name", list(FAMILIES))
def test_family_derivatives_against_complex_step(probe, name):
    idx, f, D, P = FAMILIES[name]
    rng = np.random.default_rng(100 + idx)
    n = 64
    u, p, ud, l = _points(name, n, rng)
    W = 2 * D * D + 2 * D + 2 * P
    out = _zeros((n, W))
    du, dpar, dud, dl = _dev(u), _dev(p), _dev(ud), _dev(l)          # held until the launch returns
    _check(probe.probe_family(idx, n, du.data_ptr(), dpar.data_ptr(), dud.data_ptr(), dl.data_ptr(), out.data_ptr()))
    out = out.cpu().numpy()
    worst = {}
    for i in range(n):
        o = out[i]
        fd, Jd, dJd = o[:D], o[D:D + D * D].reshape(D, D), o[D + D * D:D + 2 * D * D].reshape(D, D)
        dvd, vud, vpd = o[D + 2 * D * D:D + 2 * D * D + P], o[D + 2 * D * D + P:2 * D + 2 * D * D + P], o[2 * D + 2 * D * D + P:]
        J, F = cs_first(f, u[i], p[i], D, P)
        dJ, dF = cs_second(f, u[i], p[i], ud[i], D, P)
        fr = np.array([complex(v).real for v in f(list(u[i]), list(p[i]))])
        checks = {
            "f": _rel_err(fd, fr, np.abs(fr).max()),
            "jac": _rel_err(Jd, J, np.abs(J).max()),
            "djac": _rel_err(dJd, dJ, np.abs(dJ).max()),
            "vjp_u": _rel_err(vud, l[i] @ J, np.max(np.abs(l[i]) @ np.abs(J))),
            "vjp_p": _rel_err(vpd, l[i] @ F, np.max(np.abs(l[i]) @ np.abs(F))),
            "dvjp_p": _rel_err(dvd, l[i] @ dF, np.max(np.abs(l[i]) @ np.abs(dF))),
        }
        for k, e in checks.items():
            worst[k] = max(worst.get(k, 0.0), float(np.max(e)))
    bad = {k: v for k, v in worst.items() if not v <= 1e-14}
    assert not bad, (name, worst)


@pytest.mark.parametrize("name", list(FAMILIES))
def test_reference_hessian_is_constant(name):
    """djac(p, yd) takes no u: the right-hand sides are quadratic, so d/de J(u + e yd) is the same at every u (checked on the
    restated f; a non-quadratic family has no such djac)."""
    idx, f, D, P = FAMILIES[name]
    rng = np.random.default_rng(7 + idx)
    u, p, ud, _ = _points(name, 3, rng)
    for i in range(1, 3):
        a, A = cs_second(f, u[0], p[0], ud[0], D, P)
        b_, B = cs_second(f, u[i], p[0], ud[0], D, P)
        assert np.array_equal(a, b_)


# ------------------------------------------------------------------------------------------------------------------------
# lu_factor / lu_solve


def _lu(probe, A, b):
    n, D = A.shape[0], A.shape[1]
    ok, piv, LU, x = _zeros((n,), "i"), _zeros((n, D), "i"), _zeros((n, D, D)), _zeros((n, D))
    dA, db = _dev(A), _dev(b)
    _check(probe.probe_lu(D, n, dA.data_ptr(), db.data_ptr(), ok.data_ptr(), piv.data_ptr(), LU.data_ptr(), x.data_ptr()))
    return ok.cpu().numpy(), piv.cpu().numpy(), LU.cpu().numpy(), x.cpu().numpy()


def lu_pivots(A):
    """partial pivoting with the kernel's rule (first row of the largest |entry|, strict >), exact rational elimination"""
    D = len(A)
    M = [[Fraction(float(v)) for v in row] for row in A]
    piv = []
    for c in range(D):
        pr, mx = c, abs(M[c][c])
        for r in range(c + 1, D):
            if abs(M[r][c]) > mx:
                pr, mx = r, abs(M[r][c])
        piv.append(pr)
        if mx == 0:
            return piv, False
        M[c], M[pr] = M[pr], M[c]
        for r in range(c + 1, D):
            f = M[r][c] / M[c][c]
            M[r][c] = f
            for j in range(c + 1, D):
                M[r][j] -= f * M[c][j]
    return piv, True


def _dyadic_systems(D, n, rng):
    """A = Perm (L U): L unit lower with entries in {+-1/4, +-1/2, +-3/4}, U upper with power-of-two diagonal and integer
    entries, x integer: every step of the elimination and the substitutions is exact in fp64"""
    A, x = np.zeros((n, D, D)), np.zeros((n, D))
    for i in range(n):
        L = np.eye(D)
        for r in range(D):
            for c in range(r):
                L[r, c] = rng.choice([-0.75, -0.5, -0.25, 0.25, 0.5, 0.75])
        U = np.triu(rng.integers(-6, 7, (D, D)).astype(float), 1) + np.diag(2.0 ** rng.integers(0, 5, D) * rng.choice([-1, 1], D))
        A[i] = (L @ U)[rng.permutation(D)]
        x[i] = rng.integers(-20, 21, D)
    return A, np.einsum("nij,nj->ni", A, x), x


@pytest.mark.gpu
@pytest.mark.parametrize("D", [1, 2, 3])
def test_lu_exact_on_dyadic_systems(probe, D):
    rng = np.random.default_rng(D)
    A, b, x = _dyadic_systems(D, 200, rng)
    ok, piv, _, xd = _lu(probe, A, b)
    assert ok.all()
    assert np.array_equal(xd, x)
    for i in range(len(A)):
        assert list(piv[i]) == lu_pivots(A[i])[0], (i, A[i])


@pytest.mark.gpu
@pytest.mark.parametrize("D", [1, 2, 3])
def test_lu_pivots_and_singular_matrices(probe, D):
    cases = []       # (A, expected piv, expected ok)
    if D == 1:
        cases += [([[2.0]], [0], True), ([[-0.5]], [0], True), ([[0.0]], [0], False)]
    if D == 2:
        cases += [([[0.0, 1.0], [3.0, 2.0]], [1, 1], True),              # zero leading pivot: swap
                  ([[2.0, 1.0], [-2.0, 5.0]], [0, 1], True),             # equal magnitudes: the first row stays
                  ([[-1.0, 4.0], [1.0, 1.0]], [0, 1], True),
                  ([[1.0, 2.0], [2.0, 4.0]], [1, 1], False),             # singular: rank 1
                  ([[0.0, 1.0], [0.0, 3.0]], [0], False)]                # singular: zero column
    if D == 3:
        cases += [([[0.0, 1.0, 2.0], [0.0, 3.0, 1.0], [4.0, 1.0, 1.0]], [2, 1, 2], True),
                  ([[1.0, 2.0, 3.0], [-1.0, 1.0, 0.0], [1.0, 0.0, 2.0]], [0, 1, 2], True),      # equal magnitudes in column 0
                  ([[2.0, 0.0, 1.0], [4.0, 1.0, 1.0], [-4.0, 3.0, 2.0]], [1, 2, 2], True),
                  ([[1.0, 2.0, 3.0], [2.0, 4.0, 6.0], [1.0, 1.0, 1.0]], [1, 2, 2], False),
                  ([[1.0, 0.0, 0.0], [0.0, 0.0, 1.0], [0.0, 0.0, 2.0]], [0, 1], False)]
    A = np.array([c[0] for c in cases])
    x = np.arange(1, D + 1, dtype=float)
    b = np.einsum("nij,j->ni", A, x)
    ok, piv, _, xd = _lu(probe, A, b)
    for i, (Ai, pv, good) in enumerate(cases):
        assert lu_pivots(np.array(Ai)) == (pv, good)         # the expectation follows the kernel's rule
        assert bool(ok[i]) == good, (Ai, ok[i])
        assert list(piv[i][:len(pv)]) == pv, (Ai, piv[i])
        if good:
            assert np.abs(xd[i] - x).max() <= 4 * D * np.finfo(float).eps * np.abs(x).max() * np.linalg.cond(np.array(Ai), np.inf), (Ai, xd[i])


def robertson_w_systems(rng, hs=None, adjoint=False):
    """W = I - h d J(y, k) (forward) or I + hs d J' with hs = -h (the lambda block of the reverse solves, which step
    backwards) at points of Robertson's trajectory"""
    import mpmath as mp
    if hs is None:
        hs = np.logspace(-4, np.log10(90.0), 25)
    mats, rhs = [], []
    for h in hs:
        for _ in range(4):
            y0 = rng.uniform(0.3, 1.0)
            y1 = rng.uniform(1e-5, 4e-5)
            y = [y0, y1, 1.0 - y0 - y1]
            k = [0.04, 3e7, 1e4]
            J, _ = cs_first(f_robertson, y, k, 3, 3)
            hd = h * ROS_D
            W = np.eye(3) - hd * J.T if adjoint else np.eye(3) - hd * J      # the reverse solves: I + hs d J', hs = -h < 0
            mats.append(W)
            rhs.append(rng.standard_normal(3) * 10.0 ** rng.uniform(-3, 3))
    return np.array(mats), np.array(rhs)


def mp_solve(W, b):
    """40-digit solve of the fp64 matrix and right-hand side as given; -> (x, cond_inf)"""
    import mpmath as mp
    with mp.workdps(40):
        M = mp.matrix([[mp.mpf(float(v)) for v in row] for row in W])
        x = mp.lu_solve(M, mp.matrix([mp.mpf(float(v)) for v in b]))
        cond = mp.mnorm(M, mp.inf) * mp.mnorm(M ** -1, mp.inf)
        return np.array([float(v) for v in x]), float(cond)


@pytest.mark.gpu
@pytest.mark.parametrize("adjoint", [False, True])
def test_lu_robertson_w_against_40_digits(probe, adjoint):
    rng = np.random.default_rng(11 + adjoint)
    W, b = robertson_w_systems(rng, adjoint=adjoint)
    ok, _, _, xd = _lu(probe, W, b)
    assert ok.all()
    eps = np.finfo(float).eps
    worst, cmax = 0.0, 0.0
    for i in range(len(W)):
        x, cond = mp_solve(W[i], b[i])
        ratio = np.abs(xd[i] - x).max() / np.abs(x).max() / (cond * eps)
        worst, cmax = max(worst, ratio), max(cmax, cond)
        assert ratio <= 4 * 3, (i, ratio, cond)
    print(f"Robertson W ({'adjoint' if adjoint else 'forward'}): max cond {cmax:.3g}, max err / (cond eps) {worst:.3g}")


# ------------------------------------------------------------------------------------------------------------------------
# FwdDense<D>::eval


def dense_eval(knots, u, k1, k2, iv, t):
    """y, yd of interval iv with the kernel's operations: th = (t - ta) / h, c1 = th (1 - th) / (1 - 2d), c2 = th (th - 2d) /
    (1 - 2d), y = fma(h, fma(k1, c1, k2 c2), u), yd = fma(k1, d1, k2 d2); yd_cs = complex-step derivative of y in t"""
    ta, tb = knots[iv], knots[iv + 1]
    h = tb - ta
    th = 1.0 if h == 0.0 else (t - ta) / h
    c1, c2 = ((1 - th) * th) / IC, ((th - 2 * ROS_D) * th) / IC
    d1, d2 = (1 - 2 * th) / IC, (2 * th - 2 * ROS_D) / IC
    y = np.array([fma(h, fma(k1[j], c1, k2[j] * c2), u[j]) for j in range(len(u))])
    yd = np.array([fma(k1[j], d1, k2[j] * d2) for j in range(len(u))])
    dl = 1e-60
    if h != 0.0:
        thc = (complex(t, dl) - ta) / h
        yc = [u[j] + h * (thc * (1 - thc) / (1 - 2 * ROS_D) * k1[j] + thc * (thc - 2 * ROS_D) / (1 - 2 * ROS_D) * k2[j]) for j in range(len(u))]
        yd_cs = np.array([v.imag / dl for v in yc])
    else:               # zero-length interval: th = 1 on it, the derivative of the interpolant's bracket in th
        thc = complex(1.0, dl)
        yd_cs = np.array([(thc * (1 - thc) / (1 - 2 * ROS_D) * k1[j] + thc * (thc - 2 * ROS_D) / (1 - 2 * ROS_D) * k2[j]).imag / dl for j in range(len(u))])
    return y, yd, yd_cs


def _knot_sets():
    geo = 1e-3 * 1.7 ** np.arange(14)
    geo = np.concatenate([[0.0], geo])
    dyadic = np.arange(17) / 8.0
    repeated = np.array([0.0, 0.5, 0.5, 1.0, 1.25, 1.25, 1.25, 2.0, 2.0 + 2.0 ** -20, 3.0])
    single = np.array([0.0, 3.0])
    return [geo, dyadic, repeated, single]


def _queries(knots, rng, Q):
    """as the reverse solve makes them: downwards with several lookups per interval (t, t + h/2, t + h with continuity right,
    the quadrature nodes left), every knot exactly with both continuities, and an occasional jump upwards"""
    T, t0 = knots[-1], knots[0]
    out = []
    t = T
    while len(out) < Q and t > t0:
        hs = -min(t - t0, (T - t0) * rng.uniform(0.005, 0.15))
        out += [(t, 1), (t + 0.5 * hs, 1), (t + hs, 1), (t + 0.5 * hs, 0)]
        near = [k for k in knots if t + hs <= k <= t]
        for k in near:
            out += [(k, 1), (k, 0)]
        if rng.uniform() < 0.1:                                   # upward jump, then carry on downwards
            out += [(min(T, t + (T - t0) * rng.uniform(0.05, 0.5)), int(rng.integers(0, 2)))]
        t = t + hs
    out += [(t0, 1), (t0, 0), (T, 0), (T, 1)]
    while len(out) < Q:
        out.append((rng.uniform(t0, T), int(rng.integers(0, 2))))
    return out[:Q]


@pytest.mark.gpu
@pytest.mark.parametrize("D", [1, 2, 3])
def test_forward_dense_lookups(probe, D):
    rng = np.random.default_rng(40 + D)
    sets = _knot_sets()
    N, Q = len(sets), 400
    nmax = max(len(s) - 1 for s in sets)
    ft = np.zeros((nmax + 1, N))
    fu = np.zeros((nmax + 1, D, N))
    fk = np.zeros((nmax, 2, D, N))
    nk = np.zeros(N, dtype=np.int32)
    tq, rq = np.zeros((N, Q)), np.zeros((N, Q), dtype=np.int32)
    for i, kn in enumerate(sets):
        n = len(kn) - 1
        nk[i] = n
        ft[:n + 1, i] = kn
        fu[:n + 1, :, i] = rng.standard_normal((n + 1, D))
        fk[:n, :, :, i] = rng.standard_normal((n, 2, D)) * 3.0
        for k, (t, r) in enumerate(_queries(kn, rng, Q)):
            tq[i, k], rq[i, k] = t, r
    y, yd, iv = _zeros((N, Q, D)), _zeros((N, Q, D)), _zeros((N, Q), "i")
    ins = [_dev(a) for a in (ft, fu, fk, nk, tq, rq)]
    _check(probe.probe_dense(D, ins[0].data_ptr(), ins[1].data_ptr(), ins[2].data_ptr(), ins[3].data_ptr(), N, Q,
                             ins[4].data_ptr(), ins[5].data_ptr(), y.data_ptr(), yd.data_ptr(), iv.data_ptr()))
    y, yd, iv = y.cpu().numpy(), yd.cpu().numpy(), iv.cpu().numpy()
    for i, kn in enumerate(sets):
        n = nk[i]
        for k in range(Q):
            t, r = tq[i, k], bool(rq[i, k])
            ivr = dense_interval(kn, n, t, r)
            assert iv[i, k] == ivr, (i, k, t, r, iv[i, k], ivr)
            yr, ydr, ydc = dense_eval(kn, fu[ivr, :, i], fk[ivr, 0, :, i], fk[ivr, 1, :, i], ivr, t)
            assert np.array_equal(y[i, k], yr), (i, k, t, r, y[i, k], yr)
            assert np.array_equal(yd[i, k], ydr), (i, k, t, r, yd[i, k], ydr)
            assert np.abs(yd[i, k] - ydc).max() <= 1e-14 * max(np.abs(ydc).max(), np.abs(fk[ivr, :, :, i]).max()), (i, k, yd[i, k], ydc)


# ------------------------------------------------------------------------------------------------------------------------
# step_factor_I, tstop_snap


def step_factor_ref(e):
    q = max(e, 1e-300) ** (1.0 / 3.0) / 0.9
    return max(0.1, min(5.0, q))


def tstop_snap_ref(tn, ts):
    tol = EPS100 * max(abs(tn), abs(ts))
    return ts if abs(tn - ts) <= tol else tn


@pytest.mark.gpu
def test_step_factor_and_tstop_snap(probe):
    # EEst edges: 0, 1e-300, 1, deep in both clamps, and at the clamps' edges (0.09^3, (4.5)^3) where the clamp decides
    eest = np.array([0.0, 1e-300, 5e-324, 1e-200, 1e-12, 1e-4, 7.29e-4 * 0.999, 1.0, 91.125 * 1.001, 1e3, 1e300, np.inf])
    # tstop within 100 eps on either side: steps of one ulp around the snap boundary, at several magnitudes and signs
    tn, ts = [], []
    for s in (1.0, 100.0, 1e-3, 0.75, -2.0, 3e5):
        for k in list(range(-4, 5)) + list(range(90, 110)) + list(range(190, 210)) + [-95, -100, -101, -105, -199, -200, -201]:
            x = s
            for _ in range(abs(k)):
                x = np.nextafter(x, np.inf if k > 0 else -np.inf)
            tn.append(x)
            ts.append(s)
    n = max(len(eest), len(tn))
    e = np.resize(eest, n)
    tn, ts = np.array(tn + tn[:n - len(tn)]), np.array(ts + ts[:n - len(ts)])
    q, snap = _zeros((n,)), _zeros((n,))
    de, dtn, dts = _dev(e), _dev(tn), _dev(ts)
    _check(probe.probe_scalars(n, de.data_ptr(), q.data_ptr(), dtn.data_ptr(), dts.data_ptr(), snap.data_ptr()))
    q, snap = q.cpu().numpy(), snap.cpu().numpy()
    for i in range(n):
        assert q[i] == step_factor_ref(e[i]), (e[i], q[i], step_factor_ref(e[i]))
        assert snap[i] == tstop_snap_ref(tn[i], ts[i]), (tn[i], ts[i], snap[i])
    assert (snap == ts).sum() > 0 and (snap != ts).sum() > 0          # both sides of the boundary were visited
