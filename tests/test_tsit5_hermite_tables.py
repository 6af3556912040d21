"""The Hermite-form dense-output tables of the fixed-step Tsit5 reverse kernel (csrc/ode_tsit5.cuh, tsit5_dense_hermite),
as the library builds them for a handle (api.cu, build_tsit5_tables), through tests/csrc/tsit5_tables_probe.cu.

The kernel evaluates the forward dense output y(theta) = u_n + sum_j h b_j(theta) k_j at the 4 adjoint stage times and the
3 Gauss nodes as u_n + H01 du + h H10 k1 + h H11 k7 + theta^2 (1-theta)^2 c4 with du = u_{n+1} - u_n = sum_j h b_j k_j and
c4 = sum_j hR4[j] k_j.  Expanded over the stages, the weight of k_j must be h b_j(theta) at the theta of the direct-form
row (hBst, hBq) it replaces: this pins the Hermite identities of the Tsit5 interpolant (b_j(1) = b_j, b_j'(0) = delta_j1,
b_j'(1) = delta_j7) and the point order of the table (row 4 + g is the y-side node of Gauss point g, the theta of hBq[2 - g]).
The reference is the published factored form of b_j(theta) (Tsitouras 2011) evaluated in exact rational arithmetic: the
direct-form tables themselves round by up to ~8e-15 h (Horner on coefficients up to 47), the Hermite form by < 1e-15 h.
No GPU needed."""
import ctypes as C
import os
import subprocess
from fractions import Fraction as F

import numpy as np
import pytest

from scimlsensitivity_jl_b200 import _lib

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
CSRC = os.path.join(ROOT, "scimlsensitivity.jl_b200", "csrc")
PROBE = os.path.join(ROOT, "tests", "csrc", "tsit5_tables_probe.cu")


def b_exact(j, th):
    """Tsit5 dense-output weight b_j(theta), factored form, exact at the given (double) theta."""
    t = F(th)
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

    def get(h):
        buf = np.zeros(256)
        n = lib.probe_tsit5_tables(h, buf.ctypes.data, buf.size)
        assert n == 42 + 28 + 21 + 3 + 28 + 7, n        # hA, hBst, hBq, hGW, hHm, hR4
        o = np.cumsum([0, 42, 28, 21, 3, 28, 7])
        return {"hA": buf[o[0]:o[1]].reshape(7, 6), "hBst": buf[o[1]:o[2]].reshape(4, 7), "hBq": buf[o[2]:o[3]].reshape(3, 7),
                "hGW": buf[o[3]:o[4]], "hHm": buf[o[4]:o[5]].reshape(7, 4), "hR4": buf[o[5]:o[6]]}
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
