"""The right-hand sides of the built-in families restated in plain Python, generic over the number type (float, complex,
mpmath, bicomplex): the only model input of the Rosenbrock23 and adaptive Tsit5 probes and of the 40-digit reference, which
derive every derivative from these by differentiation (tests/test_gpu_ros23_probe.py, tests/test_gpu_ros23_reference.py,
tests/test_gpu_t5a_probe.py).  Also the stepper-independent pieces those tests share: the dense-lookup restatements,
complex-step VJPs in 40 digits, `tstop_snap`, the test problems and the LvClone plug-in."""
import os
from fractions import Fraction

import numpy as np

import mpmath as mp

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
EPS100 = 100 * 2.220446049250313e-16


def f_lv(u, p):
    return [p[0] * u[0] - p[1] * u[0] * u[1], -p[2] * u[1] + p[3] * u[0] * u[1]]


def f_lorenz(u, p):
    return [p[0] * (u[1] - u[0]), u[0] * (p[1] - u[2]) - u[1], u[0] * u[1] - p[2] * u[2]]


def f_robertson(y, k):
    return [-k[0] * y[0] + k[2] * y[1] * y[2], k[0] * y[0] - k[1] * y[1] * y[1] - k[2] * y[1] * y[2], k[1] * y[1] * y[1]]


def f_ball(u, p):
    return [u[1] + 0 * p[0], -p[0] + 0 * u[0]]


def f_relax(u, p):
    return [p[0] - u[0]]


def fma(a, b, c):
    """a * b + c rounded once"""
    return float(Fraction(a) * Fraction(b) + Fraction(c))


def dense_interval(knots, n, t, right):
    """the interval the cursor search stops on, from a scan of all knots: right = largest idx with T(idx) <= t, left =
    (smallest idx >= 1 with T(idx) >= t) - 1, clamped to [0, n - 1]"""
    if right:
        iv = max([k for k in range(n) if knots[k] <= t], default=0)
    else:
        iv = max([k for k in range(n) if k == 0 or knots[k] < t], default=0)
    return min(max(iv, 0), n - 1)


def tstop_snap(tn, ts):
    """a step end within 100 eps of a tstop lands on it (ros23.cuh::tstop_snap)"""
    return ts if abs(tn - ts) <= EPS100 * max(abs(tn), abs(ts)) else tn


def vjp_p(f, y, p, l):
    """(df/dp)' l by complex steps of l' f(y, p)"""
    dl = mp.mpf("1e-30")
    out = []
    for q in range(len(p)):
        pc = [mp.mpc(v) for v in p]
        pc[q] += mp.mpc(0, dl)
        out.append(mp.im(sum(l[r] * v for r, v in enumerate(f(y, pc)))) / dl)
    return out


def vjp_u(f, y, p, l):
    """(df/du)' l by complex steps of l' f(y, p)"""
    dl = mp.mpf("1e-30")
    out = []
    for c in range(len(y)):
        yc = [mp.mpc(v) for v in y]
        yc[c] += mp.mpc(0, dl)
        out.append(mp.im(sum(l[r] * v for r, v in enumerate(f(yc, p)))) / dl)
    return out


def problem(family, N, shared_p):
    """-> (t0, T, saveat, u0[D][N], p[P] or [P][N])"""
    rng = np.random.default_rng({"lv": 1, "lv_clone": 1, "lorenz": 2, "robertson": 3}[family])
    if family in ("lv", "lv_clone"):
        T, u0, p = 2.0, np.exp(0.1 * rng.standard_normal((2, N))), np.array([1.5, 1.0, 3.0, 1.0])
        saveat = np.linspace(0.25, T, 8)
    elif family == "lorenz":
        T, u0, p = 0.5, np.array([1.0, 0.0, 0.0])[:, None] + 0.1 * rng.standard_normal((3, N)), np.array([10.0, 28.0, 8.0 / 3.0])
        saveat = np.linspace(0.05, T, 10)
    else:
        T, u0, p = 10.0, np.repeat(np.array([[1.0], [0.0], [0.0]]), N, 1), np.array([0.04, 3e7, 1e4])
        saveat = np.logspace(-2, 1, 6)
    if not shared_p:
        p = p[:, None] * np.exp(0.05 * rng.standard_normal((len(p), N)))
    return 0.0, T, saveat, u0, p


def register_lv_clone():
    """the LvClone plug-in example (examples/lv_clone_family.cuh), built next to it unless a loadable build is there"""
    import scimlsensitivity_jl_b200 as b
    so = os.path.join(ROOT, "examples", "libb200fam_lv_clone.so")
    if os.path.exists(so):
        try:
            return b.register_family(so)
        except b.B200AdjError:
            os.remove(so)
    return b.register_family(b.build_family_plugin(os.path.join(ROOT, "examples", "lv_clone_family.cuh"), "LvClone", "lv_clone", out=so, has_jac=True))
