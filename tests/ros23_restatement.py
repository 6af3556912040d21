"""The right-hand sides of the built-in families restated in plain Python, generic over the number type (float, complex,
mpmath, bicomplex): the only model input of the Rosenbrock23 and adaptive Tsit5 probes and of the 40-digit reference, which
derive every derivative from these by differentiation (tests/test_gpu_ros23_probe.py, tests/test_gpu_ros23_reference.py,
tests/test_gpu_t5a_probe.py).  Also the stepper-independent pieces those tests share: the dense-lookup restatements,
complex-step VJPs in 40 digits, `tstop_snap`, the test problems, the LvClone plug-in and the Tsit5 tableau as published
(tests/test_tsit5_hermite_tables.py, tests/test_gpu_t5a_probe.py, tests/test_gpu_fixed_probe.py,
tests/test_gpu_fixed_reference.py)."""
import os
from fractions import Fraction

import numpy as np

import mpmath as mp

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
EPS100 = 100 * 2.220446049250313e-16

# Tsit5 (Tsitouras 2011), as published: A (row 6 = b, b_7 = 0), c, and the embedded error weights btilde = b - bhat
A_TXT = [[], ["0.161"], ["-0.008480655492356989", "0.335480655492357"],
         ["2.897153057105493", "-6.359448489975075", "4.3622954328695815"],
         ["5.325864828439257", "-11.748883564062828", "7.4955393428898365", "-0.09249506636175525"],
         ["5.86145544294642", "-12.92096931784711", "8.159367898576159", "-0.071584973281401", "-0.028269050394068383"],
         ["0.09646076681806523", "0.01", "0.4798896504144996", "1.379008574103742", "-3.290069515436081", "2.324710524099774"]]
C_TXT = ["0.0", "0.161", "0.327", "0.9", "0.9800255409045097", "1.0", "1.0"]
BT_TXT = ["-0.00178001105222577714", "-0.0008164344596567469", "0.007880878010261995", "-0.1447110071732629",
          "0.5823571654525552", "-0.45808210592918697", "0.015151515151515152"]


def b_exact(j, th):
    """Tsit5 dense-output weight b_j(theta), the published factored form, exact at the given theta (float or Fraction)"""
    t = Fraction(th)
    F = Fraction
    if j == 0:
        return F("-1.0530884977290216") * t * (t - F("1.3299890189751412")) * (t * t - F("1.4364028541716351") * t + F("0.7139816917074209"))
    if j in (1, 2):
        c, s, w = {1: ("0.1017", "2.1966568338249754", "1.2949852507374631"),
                   2: ("2.490627285651252793", "2.38535645472061657", "1.57803468208092486")}[j]
        return F(c) * t * t * (t * t - F(s) * t + F(w))
    c, r1, r2 = {3: ("-16.54810288924490272", "1.21712927295533244", "0.61620406037800089"),
                 4: ("47.37952196281928122", "1.203071208372362603", "0.658047292653547382"),
                 5: ("-34.87065786149660974", "1.2", "0.666666666666666667"),
                 6: ("2.5", "1.0", "0.6")}[j]
    return F(c) * (t - F(r1)) * (t - F(r2)) * t * t


def _r_exact():
    """R[j][m]: b_j(theta) = sum_m R[j][m] theta^(m+1), from the factored b_exact at theta = 1..4 (exact rationals)"""
    R = []
    for j in range(7):
        M = [[Fraction(th) ** (m + 1) for m in range(4)] + [b_exact(j, th)] for th in (1, 2, 3, 4)]
        for c in range(4):
            for r in range(c + 1, 4):
                f = M[r][c] / M[c][c]
                M[r] = [M[r][k] - f * M[c][k] for k in range(5)]
        x = [Fraction(0)] * 4
        for c in range(3, -1, -1):
            x[c] = (M[c][4] - sum(M[c][k] * x[k] for k in range(c + 1, 4))) / M[c][c]
        R.append(x)
    return R


R_EXACT = _r_exact()


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
