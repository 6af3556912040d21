"""The folded Hermite point table of the fixed-step Tsit5 reverse kernel (OdeRevArgsT::hHf; api.cu, build_hermite_folded),
through tests/csrc/tsit5_folded_probe.cu and tests/csrc/tsit5_tables_probe.cu.

The kernel forms the dense output at the 4 adjoint stage times and the 3 Gauss nodes as
    y = u_n + alpha du + beta k1 + gamma k7 + G c4'',   c4'' = sum_{j=1..4} w_j k_j
(csrc/ode_tsit5.cuh, tsit5_hermite_c4_du and tsit5_dense_hermite): the Hermite form u_n + H01 du + h H10 k1 + h H11 k7 + G c4
with c4's k6 eliminated through du = sum_{j<6} h b_j k_j (w = hC4u, build_c4_du_weights) and its w_0 k1, w_5 du and w_6 k7
terms folded into the point weights: alpha = H01 + G w_5, beta = h H10 + G w_0, gamma = h H11 + G w_6, G = theta^2 (1-theta)^2.
The Gauss block takes lambda from the adjoint step's own dense output in the same form, node g from row 6 - g.

Pinned here, in exact rational arithmetic:
* every entry of hHf against the exact fold at the library's own theta, b and theta^4 coefficients, to half an ulp (a double
  evaluation of the same formulas is off by up to 24 ulps);
* expanded over the stages, each row's weight of k_j is h b_j(theta) of the published factored form (Tsitouras 2011) at the
  row's theta, and agrees with the direct-form row it stands for (hBst, hBq[2 - g]);
* the lambda rows of the Gauss block: row 6 - g sits at the theta of hBq[g], the y-side row 4 + g at 1 - that theta (the
  same time), and row 6 - g expands to hBq[g];
* the fp32 weights (hC4u and hHf as the fp32 reverse pass receives them): each the float nearest its fp64 value, and the
  expansion holds at float rounding.
No GPU needed."""
import ctypes as C
import os
import subprocess
from fractions import Fraction as F

import numpy as np
import pytest

from scimlsensitivity_jl_b200 import _lib
from ros23_restatement import b_exact

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
CSRC = os.path.join(ROOT, "scimlsensitivity.jl_b200", "csrc")
PROBES = [os.path.join(ROOT, "tests", "csrc", s) for s in ("tsit5_folded_probe.cu", "tsit5_tables_probe.cu")]
EPS32 = 2.0 ** -23
HS = [0.01, 1e-3, 0.37, 1.0]


@pytest.fixture(scope="module")
def probe(tmp_path_factory):
    """the two probes linked against the library, built outside the source tree"""
    _lib.build()
    pkg = os.path.dirname(_lib.LIB_PATH)
    so = str(tmp_path_factory.mktemp("tsit5_folded_probe") / "libtsit5_folded_probe.so")
    cmd = [_lib.nvcc_path(), "-gencode", "arch=compute_90a,code=sm_90a", "-O3", "-std=c++17", "-I", CSRC,
           "-Xcompiler", "-fPIC", "-shared", *PROBES, "-o", so, "-L", pkg, "-lb200adj", "-Xlinker", "-rpath," + pkg]
    res = subprocess.run(cmd, capture_output=True, text=True)
    assert res.returncode == 0, res.stdout[-3000:] + res.stderr[-3000:]
    lib = C.CDLL(so)
    lib.probe_hermite_folded.argtypes = [C.c_double, C.c_void_p]
    lib.probe_hermite_thetas.argtypes = [C.c_void_p]
    lib.probe_hermite_weights_f32.argtypes = [C.c_double, C.c_void_p, C.c_void_p]
    lib.probe_tsit5_tables.argtypes = [C.c_double, C.c_void_p, C.c_int]
    lib.probe_tsit5_tables.restype = C.c_int
    lib.probe_tsit5_tables_f32.argtypes = [C.c_double, C.c_void_p, C.c_int]
    lib.probe_tsit5_tables_f32.restype = C.c_int
    lib.probe_c4_du_weights.argtypes = [C.c_double, C.c_void_p]
    lib.probe_tsit5_rpoly.argtypes = [C.c_void_p]

    class P:
        @staticmethod
        def folded(h):
            hf = np.zeros((7, 4))
            lib.probe_hermite_folded(h, hf.ctypes.data)
            return hf

        @staticmethod
        def thetas():
            th = np.zeros(7)
            lib.probe_hermite_thetas(th.ctypes.data)
            return th

        @staticmethod
        def f32(h):
            c4u, hf = np.zeros(7, dtype=np.float32), np.zeros((7, 4), dtype=np.float32)
            lib.probe_hermite_weights_f32(h, c4u.ctypes.data, hf.ctypes.data)
            return c4u, hf

        @staticmethod
        def tables(h, f32=False):
            """hA[6] (h b), hBst and hBq of the table struct (layout pinned by test_tsit5_hermite_tables.py)"""
            buf = np.zeros(256, dtype=np.float32 if f32 else np.float64)
            n = (lib.probe_tsit5_tables_f32 if f32 else lib.probe_tsit5_tables)(h, buf.ctypes.data, buf.size)
            assert n == 129, n
            return {"hb": buf[36:42], "hBst": buf[42:70].reshape(4, 7), "hBq": buf[70:91].reshape(3, 7)}

        @staticmethod
        def c4u(h):
            w = np.zeros(7)
            lib.probe_c4_du_weights(h, w.ctypes.data)
            return w

        @staticmethod
        def rpoly():
            R = np.zeros((7, 4))
            lib.probe_tsit5_rpoly(R.ctypes.data)
            return R
    return P


def _ulp(x):
    return F(float(np.spacing(abs(float(x)))))


def _fold(h, x, b, r4, G=None):
    """(alpha, beta, gamma, G) at theta x from b_j and the theta^4 coefficients r4_j (all exact rationals); h exact"""
    x = F(x)
    if G is None:
        G = x * x * (1 - x) ** 2
    w0, w5, w6 = h * (r4[0] - r4[5] * b[0] / b[5]), r4[5] / b[5], h * r4[6]
    return [3 * x ** 2 - 2 * x ** 3 + G * w5, h * (x - 2 * x ** 2 + x ** 3) + G * w0, h * (x ** 3 - x ** 2) + G * w6, G]


def _expand(row, hb, w):
    """the weights of k_1..k_7 in u_n + alpha du + beta k1 + gamma k7 + G sum_{j=1..4} w_j k_j with du = sum_{j<6} hb_j k_j"""
    al, be, ga, G = (F(float(v)) for v in row)
    out = [al * F(float(hb[j])) for j in range(6)] + [F(0)]
    out[0] += be
    out[6] += ga
    for j in range(1, 5):
        out[j] += G * F(float(w[j]))
    return out


def _exact_row(h, th):
    return [F(h) * b_exact(j, th) for j in range(7)]


@pytest.mark.parametrize("h", HS)
def test_folded_table_is_the_exact_fold(probe, h):
    """each entry of hHf within half an ulp of the fold at the library's own theta, b = A[6] and theta^4 coefficients R[:, 3]
    (exact rationals); the same formulas evaluated in double leave some entry more than 8 ulps off (15 to 24 at these h):
    the long double is needed"""
    hf, th = probe.folded(h), probe.thetas()
    b = [F(float(v)) for v in probe.tables(1.0)["hb"]]           # h = 1: hA[6] is b itself
    R = probe.rpoly()
    r4 = [F(R[j][3]) for j in range(7)]
    worst_dbl = 0.0
    for r in range(7):
        ex = _fold(F(h), th[r], b, r4)
        for m in range(4):
            assert abs(F(hf[r][m]) - ex[m]) <= _ulp(ex[m]) / 2 * F(1001, 1000), (r, m, hf[r][m], float(ex[m]))
        # the same in double: G * w_5 (up to 15/16) against H01, G * w_0 against h H10
        x, bd, rd = float(th[r]), [float(v) for v in b], [float(v) for v in r4]
        G = x * x * (1.0 - x) * (1.0 - x)
        w0, w5, w6 = h * (rd[0] - rd[5] * bd[0] / bd[5]), rd[5] / bd[5], h * rd[6]
        dbl = [3.0 * x * x - 2.0 * x ** 3 + G * w5, h * (x - 2.0 * x * x + x ** 3) + G * w0, h * (x ** 3 - x * x) + G * w6, G]
        worst_dbl = max(worst_dbl, max(float(abs(F(dbl[m]) - ex[m]) / _ulp(ex[m])) for m in range(4)))
    assert worst_dbl > 8, worst_dbl


@pytest.mark.parametrize("h", HS)
def test_folded_points_are_the_dense_output(probe, h):
    """u_n + alpha du + beta k1 + gamma k7 + G c4'' expanded over the stages (du through the library's own h b, c4'' through
    hC4u): the weight of k_j is h b_j(theta) at the row's theta, to 1e-15 h, at all 7 points; and the direct-form row the
    point replaces (hBst[r], r < 4; hBq[2 - g] at row 4 + g) agrees to its own rounding (1e-14 h)"""
    hf, th, t, w = probe.folded(h), probe.thetas(), probe.tables(h), probe.c4u(h)
    direct = np.vstack([t["hBst"], t["hBq"][::-1]])
    for r in range(7):
        got, ex = _expand(hf[r], t["hb"], w), _exact_row(h, th[r])
        err = max(abs(float(got[j] - ex[j])) for j in range(7))
        assert err <= 1e-15 * h, (r, err / h)
        assert np.abs(direct[r] - np.array([float(v) for v in got])).max() <= 1e-14 * h, r


@pytest.mark.parametrize("h", HS)
def test_lambda_rows_of_the_gauss_nodes(probe, h):
    """Gauss node g takes lambda at theta_q[g] of the adjoint step (direct form: hBq[g]) from row 6 - g, and y at the
    forward theta 1 - theta_q[g] from row 4 + g: row 6 - g has the theta of hBq[g], the two theta of node g add up to 1
    (the same time t_n + theta h = t_{n+1} - theta_q h) to an ulp, and row 6 - g expanded over the stages is hBq[g]"""
    hf, th, t, w = probe.folded(h), probe.thetas(), probe.tables(h), probe.c4u(h)
    a = np.sqrt(0.6)
    thq = [0.5 * (1.0 - a), 0.5, 0.5 * (1.0 + a)]
    for g in range(3):
        assert th[6 - g] == thq[g], (g, th[6 - g], thq[g])
        assert abs(F(th[4 + g]) + F(th[6 - g]) - 1) <= F(2.0 ** -53), g
        got = _expand(hf[6 - g], t["hb"], w)
        ex = _exact_row(h, thq[g])
        assert max(abs(float(got[j] - ex[j])) for j in range(7)) <= 1e-15 * h, g
        assert np.abs(t["hBq"][g] - np.array([float(v) for v in got])).max() <= 1e-14 * h, g


@pytest.mark.parametrize("h", HS)
def test_fp32_folded_weights(probe, h):
    """the fp32 reverse pass receives hC4u and hHf each rounded once from fp64, and with the fp32 h b of cast_tables the
    expansion gives h b_j(theta) to float rounding: 4 eps32 times the magnitudes of the terms"""
    c4u32, hf32 = probe.f32(h)
    assert np.array_equal(c4u32, probe.c4u(h).astype(np.float32))
    assert np.array_equal(hf32, probe.folded(h).astype(np.float32))
    th, hb32 = probe.thetas(), probe.tables(h, f32=True)["hb"]
    for r in range(7):
        got, ex = _expand(hf32[r], hb32, c4u32), _exact_row(h, th[r])
        al, be, ga, G = (abs(float(v)) for v in hf32[r])
        mag = [al * abs(float(hb32[j])) for j in range(6)] + [0.0]
        mag[0] += be
        mag[6] += ga
        for j in range(1, 5):
            mag[j] += G * abs(float(c4u32[j]))
        for j in range(7):
            assert abs(float(got[j] - ex[j])) <= 4 * EPS32 * mag[j] + 1e-300, (r, j, float(got[j] - ex[j]), mag[j])
