"""The Hermite-form dense-output tables of the fixed-step Tsit5 reverse kernel (csrc/ode_tsit5.cuh, tsit5_dense_hermite),
as the library builds them for a handle (api.cu, build_tsit5_tables), through tests/csrc/tsit5_tables_probe.cu.

The kernel evaluates the forward dense output y(theta) = u_n + sum_j h b_j(theta) k_j at the 4 adjoint stage times and the
3 Gauss nodes as u_n + H01 du + h H10 k1 + h H11 k7 + theta^2 (1-theta)^2 c4 with du = u_{n+1} - u_n = sum_j h b_j k_j and
c4 = sum_j hR4[j] k_j.  Expanded over the stages, the weight of k_j must be h b_j(theta) at the theta of the direct-form
row (hBst, hBq) it replaces: this pins the Hermite identities of the Tsit5 interpolant (b_j(1) = b_j, b_j'(0) = delta_j1,
b_j'(1) = delta_j7) and the point order of the table (row 4 + g is the y-side node of Gauss point g, the theta of hBq[2 - g]).
The reference is the published factored form of b_j(theta) (Tsitouras 2011) evaluated in exact rational arithmetic: the
direct-form tables themselves round by up to ~8e-15 h (Horner on coefficients up to 47), the Hermite form by < 1e-15 h.

Also pinned here, against the published decimal strings in exact rationals: the stage rows hA (h A to two ulps: the
16-17 digit strings leave the library's double one ulp from the string's nearest double at most), the Gauss weights hGW,
the dense-output polynomials Rpoly of the GaussKronrod step (tsit5_weights), the c4-from-du weights hC4u
(build_c4_du_weights: the Hermite c4 with k6 eliminated through du) in fp64 and in the float cast the fp32 reverse pass
receives, and the fp32 tables as cast_tables hands them over.  No GPU needed."""
import ctypes as C
import os
import subprocess
from fractions import Fraction as F

import numpy as np
import pytest

from scimlsensitivity_jl_b200 import _lib
from ros23_restatement import A_TXT, R_EXACT, b_exact

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
CSRC = os.path.join(ROOT, "scimlsensitivity.jl_b200", "csrc")
PROBE = os.path.join(ROOT, "tests", "csrc", "tsit5_tables_probe.cu")


@pytest.fixture(scope="module")
def tables(tmp_path_factory):
    """tsit5_tables_probe.cu linked against the library, built outside the source tree."""
    _lib.build()
    pkg = os.path.dirname(_lib.LIB_PATH)
    so = str(tmp_path_factory.mktemp("tsit5_tables_probe") / "libtsit5_tables_probe.so")
    cmd = [_lib.nvcc_path(), "-gencode", "arch=compute_90a,code=sm_90a", "-O3", "-std=c++17", "-I", CSRC,
           "-Xcompiler", "-fPIC", "-shared", PROBE, "-o", so, "-L", pkg, "-lb200adj", "-Xlinker", "-rpath," + pkg]
    res = subprocess.run(cmd, capture_output=True, text=True)
    assert res.returncode == 0, res.stdout[-3000:] + res.stderr[-3000:]
    lib = C.CDLL(so)
    lib.probe_tsit5_tables.argtypes = [C.c_double, C.c_void_p, C.c_int]
    lib.probe_tsit5_tables.restype = C.c_int
    lib.probe_tsit5_tables_f32.argtypes = [C.c_double, C.c_void_p, C.c_int]
    lib.probe_tsit5_tables_f32.restype = C.c_int
    lib.probe_c4_du_weights.argtypes = [C.c_double, C.c_void_p]
    lib.probe_tsit5_rpoly.argtypes = [C.c_void_p]

    def get(h, f32=False):
        buf = np.zeros(256, dtype=np.float32 if f32 else np.float64)
        n = (lib.probe_tsit5_tables_f32 if f32 else lib.probe_tsit5_tables)(h, buf.ctypes.data, buf.size)
        assert n == 42 + 28 + 21 + 3 + 28 + 7, n        # hA, hBst, hBq, hGW, hHm, hR4
        o = np.cumsum([0, 42, 28, 21, 3, 28, 7])
        return {"hA": buf[o[0]:o[1]].reshape(7, 6), "hBst": buf[o[1]:o[2]].reshape(4, 7), "hBq": buf[o[2]:o[3]].reshape(3, 7),
                "hGW": buf[o[3]:o[4]], "hHm": buf[o[4]:o[5]].reshape(7, 4), "hR4": buf[o[5]:o[6]]}

    def c4u(h):
        w = np.zeros(7)
        lib.probe_c4_du_weights(h, w.ctypes.data)
        return w

    def rpoly():
        R = np.zeros((7, 4))
        lib.probe_tsit5_rpoly(R.ctypes.data)
        return R
    get.c4u, get.rpoly = c4u, rpoly
    return get


@pytest.mark.parametrize("h", [0.01, 1e-3, 0.37])
def test_hermite_weights_are_the_dense_output_weights(tables, h):
    t = tables(h)
    c = [0.161, 0.327, 0.9, 0.9800255409045097]
    a = np.sqrt(0.6)
    thq = [0.5 * (1.0 - a), 0.5, 0.5 * (1.0 + a)]
    thetas = [1.0 - ci for ci in c] + [thq[2], thq[1], thq[0]]
    direct = np.vstack([t["hBst"], t["hBq"][::-1]])     # the rows the Hermite points replace: hBst, then hBq[2 - g]
    hb = np.append(t["hA"][6], 0.0)                     # du = sum_j h b_j k_j (b_7 = 0)
    for r, th in enumerate(thetas):
        exact = np.array([float(F(h) * b_exact(j, th)) for j in range(7)])
        assert np.abs(direct[r] - exact).max() <= 1e-14 * h, r       # the row's theta is this point's theta
        H01, hH10, hH11, B = t["hHm"][r]
        w = H01 * hb + B * t["hR4"]
        w[0] += hH10
        w[6] += hH11
        assert np.abs(w - exact).max() <= 1e-15 * h, (r, w - exact)


def _ulp(x):
    return F(float(np.spacing(abs(float(x)))))


def _ulp32(x):
    return F(float(np.spacing(np.float32(abs(float(x))))))


HS = [0.01, 1e-3, 0.37, 1.0]


@pytest.mark.parametrize("h", HS)
def test_stage_rows_and_gauss_weights(tables, h):
    """hA[s][j] = h A[s][j] (rows 1..6, zero above the diagonal) and hGW = (h/2) (5/9, 8/9, 5/9)"""
    t = tables(h)
    for s in range(1, 7):
        for j in range(6):
            if j >= s:
                assert t["hA"][s][j] == 0.0, (s, j)
                continue
            exact = F(h) * F(A_TXT[s][j])
            assert abs(F(t["hA"][s][j]) - exact) <= 2 * _ulp(t["hA"][s][j]), (s, j, t["hA"][s][j], float(exact))
    for g, wq in enumerate((F(5, 9), F(8, 9), F(5, 9))):
        assert abs(F(t["hGW"][g]) - F(h) / 2 * wq) <= _ulp(t["hGW"][g]), (g, t["hGW"][g])


def test_dense_output_polynomials(tables):
    """Rpoly (the GaussKronrod step's dense output, and the QuadratureAdjoint kernel's) is the expansion of the published
    factored b_j(theta), each coefficient rounded once, and reproduces b_j(theta) on [0, 1]"""
    R = tables.rpoly()
    for j in range(7):
        for m in range(4):
            assert abs(F(R[j][m]) - R_EXACT[j][m]) <= _ulp(R[j][m]) / 2 * F(1001, 1000), (j, m, R[j][m], float(R_EXACT[j][m]))
        for th in np.linspace(0.0, 1.0, 41):
            got = sum(F(R[j][m]) * F(th) ** (m + 1) for m in range(4))
            mag = sum(abs(F(R[j][m])) * F(th) ** (m + 1) for m in range(4))
            assert abs(got - b_exact(j, th)) <= F(2.3e-16) * mag, (j, th)


def _c4u_exact(h, A6, R):
    """the weights of tsit5_hermite_c4_du, exact on the library's own doubles: b = A6 (row 6 of the stage table) and R4 =
    R[:, 3]; w_j = h (R4_j - R4_5 b_j / b_6) (j < 5), w_5 = R4_5 / b_6, w_6 = h R4_6"""
    b, r = [F(v) for v in A6], [F(R[j][3]) for j in range(7)]
    return [F(h) * (r[j] - r[5] * b[j] / b[5]) for j in range(5)] + [r[5] / b[5], F(h) * r[6]]


def _c4u_in_double(h, A6, R):
    """build_c4_du_weights evaluated in double: what the long double evaluation guards against"""
    b6, r6 = float(A6[5]), float(R[5][3])
    return [h * (float(R[j][3]) - r6 * float(A6[j]) / b6) for j in range(5)] + [r6 / b6, h * float(R[6][3])]


@pytest.mark.parametrize("h", HS)
def test_c4_from_du_weights(tables, h):
    """hC4u keeps c4 = sum_j hR4_j k_j once k6 is eliminated through du = sum_{j<6} h b_j k_j:
    w_j + w_5 h b_j = h R4_j (j < 5), w_5 h b_6 = h R4_5, w_6 = h R4_6, each to one ulp of the weights that enter; and each
    weight within one ulp of the exact solution on the library's own b and R4.  The weights cancel (w_4 = -1.97 h from
    terms of 47 h and 49 h), so an evaluation in double misses the second bound: the test sees the long double."""
    w, R, A6 = tables.c4u(h), tables.rpoly(), tables(1.0)["hA"][6]     # h = 1: the stage table is A itself
    t = tables(h)
    hb, hr4 = [F(h) * F(v) for v in A6], [F(h) * F(R[j][3]) for j in range(7)]
    for j in range(5):
        res = F(w[j]) + F(w[5]) * hb[j] - hr4[j]
        assert abs(res) <= _ulp(w[j]) + _ulp(w[5]) * abs(hb[j]), (j, float(res))
    assert abs(F(w[5]) * hb[5] - hr4[5]) <= _ulp(w[5]) * abs(hb[5])
    assert w[6] == t["hR4"][6] and F(w[6]) == F(np.float64(h) * np.float64(R[6][3]))
    ex = _c4u_exact(h, A6, R)
    for j in range(7):
        assert abs(F(w[j]) - ex[j]) <= _ulp(w[j]), (j, w[j], float(ex[j]))
    dbl = _c4u_in_double(h, A6, R)
    assert max(abs(F(dbl[j]) - ex[j]) / _ulp(ex[j]) for j in range(7)) > 1


@pytest.mark.parametrize("h", HS)
def test_fp32_tables_and_c4_weights(tables, h):
    """The fp32 reverse pass receives cast_tables(h) and (float) hC4u: every entry the float nearest its fp64 value, and the
    c4 identities above hold at float rounding"""
    t, t32 = tables(h), tables(h, f32=True)
    for k in t:
        assert np.array_equal(t32[k], t[k].astype(np.float32)), k
    w32 = tables.c4u(h).astype(np.float32)
    R, A6 = tables.rpoly(), tables(1.0)["hA"][6]
    ex = _c4u_exact(h, A6, R)
    for j in range(7):
        assert abs(F(float(w32[j])) - ex[j]) <= _ulp32(w32[j]) / 2 + _ulp(ex[j]), (j, w32[j], float(ex[j]))
    hb, hr4 = t32["hA"][6], t32["hR4"]
    for j in range(5):
        res = F(float(w32[j])) + F(float(w32[5])) * F(float(hb[j])) - F(float(hr4[j]))
        bound = _ulp32(w32[j]) + _ulp32(w32[5]) * abs(F(float(hb[j]))) + abs(F(float(w32[5]))) * _ulp32(hb[j]) + _ulp32(hr4[j])
        assert abs(res) <= bound, (j, float(res), float(bound))
    res = F(float(w32[5])) * F(float(hb[5])) - F(float(hr4[5]))
    assert abs(res) <= _ulp32(w32[5]) * abs(F(float(hb[5]))) + abs(F(float(w32[5]))) * _ulp32(hb[5]) + _ulp32(hr4[5])
    assert w32[6] == hr4[6]
