"""The adaptive Tsit5 framework (csrc/tsit5_adaptive.cuh) step by step, through tests/csrc/t5a_probe.cu: the production code
called unchanged, its dense solutions read back from a handle.

* `T5Dense<D>::eval`, the reverse pass's lookup of the forward solution (two record buffers per thread in shared memory, a
  bulk-copy prefetch of the interval below, the swap at a knot, the cursor search after a jump, the `holds()` continuity
  rule), on synthetic member-major records: the interval as an integer against a scan of all knots, y bitwise against the
  kernel's fused multiply-adds restated in exact rationals.  Block sizes 32, 64 and 128; every lane of a warp has its own
  knot count and query walk; the member count is not a multiple of the block.
* Every record a forward pass stores (LV, Lorenz, Robertson with mild rates, the LvClone plug-in; shared and per-member p;
  tolerances 1e-6 to 1e-10; the constant-step dense mode; 64 members of the 65 536-member C1 ensemble): the seven stages
  recomputed in 40 digits from the record's own u_n, t_n and h; c0..c3 against sum_s R[s][m] k_s with R from the published
  factored b_j(theta) (to 1e-14 of sum |R k|); the next record's u against u_n + h sum b k; the fields t_n, t_{n+1}, h,
  1/h, the zero padding and the terminal record bitwise.
* Every controller decision of the forward pass: attempt, reject, ..., accept replayed with the PI controller's formulas
  (beta1 = 7/50, beta2 = 2/25, gamma = 0.9, q in [1/10, 5], the rejection divisor min(5, q11 / 0.9), qold = max(EEst, 1e-4))
  and the clip to t1 within 100 eps, the estimate in 40 digits.  Under the constant step every h is dt.
* Every reverse step QuadratureAdjoint stores: the seven adjoint stages in 40 digits with y from the forward records
  (right-continuous lookup), the next record's z = z + h sum b k plus the loss jump at a save time, rend = t + h bitwise,
  and the reverse controller replay with `tstop_snap` and the clip to the save times.

The replays compare step sizes on the scale of what fp64 can decide: the kernel's estimate carries the rounding of its
fp64 stages, which the embedded difference magnifies (~1e-7 relative at tolerance 1e-10), and q = EEst^(7/50) / qold^(2/25)
passes it on; the bound per decision is 0.22 times that rounding (estimated from an fp64 evaluation of the same step) plus
a few ulps of t.  Every decision is asserted to lie more than max(1e-6, that rounding) from EEst = 1.

The remaining `holds()` of the lookup only gates the fast paths: a stricter rule still lands on the right interval through the
cursor search, with the same y, and only the record buffer it reads from tells the two apart.  So the probe also reports
that buffer, against a restatement of the lookup's buffer state machine (`dense_walk`).

Observed on an H100 SXM (700 W), largest error as a share of its bound: c0..c3 0.023, next u 0.31, reverse stages 0.36, next
z 0.015, accepted step against the replay 0.064; every reverse run accepts steps with EEst < 1e-4 (5 to 8 per run), so
qold's floor is exercised.  The module took 77 s there, 43 s of it the 40-digit replay of the 64 sampled C1 members.
Mutants of tsit5_adaptive.cuh, each failing these tests there: `holds()` right continuity `ta <= t` -> `ta < t` (the
lookup's buffer), the reverse `qold = fmax(EEst, 1e-4)` -> `EEst` (the three adaptive QuadratureAdjoint runs), the
rejection divisor `fmin(5, q11 / 0.9)` -> `q` and the error norm's `fmax(|z|, |zn|)` -> `|zn|` (the forward replays, the
C1 members and the reverse runs).  Of these, test_gpu_parity_tsit5_adaptive.py fails only on the error-norm mutant.
"""
import ctypes as C
import os
import subprocess
from fractions import Fraction

import numpy as np
import pytest

import mpmath as mp

from scimlsensitivity_jl_b200 import _lib
from ros23_restatement import (A_TXT, BT_TXT, C_TXT, EPS100, R_EXACT, b_exact, dense_interval, f_lorenz, f_lv, f_robertson, fma, problem,
                               register_lv_clone, tstop_snap, vjp_u)

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
CSRC = os.path.join(ROOT, "scimlsensitivity.jl_b200", "csrc")
PROBE = os.path.join(ROOT, "tests", "csrc", "t5a_probe.cu")
EPS = 2.220446049250313e-16
DPS = 40

C64 = [float(c) for c in C_TXT]
FAMS = {"lv": (f_lv, 2, 4), "lv_clone": (f_lv, 2, 4), "lorenz": (f_lorenz, 3, 3), "robertson": (f_robertson, 3, 3)}


class Tab:
    """the tableau in 40 digits (mpf) and in fp64 (float)"""

    def __init__(self, conv):
        self.A = [[conv(v) for v in row] for row in A_TXT]
        self.BT = [conv(v) for v in BT_TXT]
        self.R = [[conv(v) if conv is float else mp.mpf(v.numerator) / v.denominator for v in row] for row in R_EXACT]


@pytest.fixture(scope="session")
def t5a_probe_so(tmp_path_factory):
    """t5a_probe.cu built with the library's nvcc flags, once per session, outside the source tree."""
    so = str(tmp_path_factory.mktemp("t5a_probe") / "libt5a_probe.so")
    cmd = [_lib.nvcc_path(), "-gencode", "arch=compute_90a,code=sm_90a", "-O3", "-std=c++17", "-I", CSRC,
           "-Xcompiler", "-fPIC", "-shared", PROBE, "-o", so]
    res = subprocess.run(cmd, capture_output=True, text=True)
    assert res.returncode == 0, res.stdout[-3000:] + res.stderr[-3000:]
    return so


def test_t5a_probe_compiles_for_sm90a(t5a_probe_so):
    """No GPU needed: a header change that breaks the probes fails here."""
    lib = C.CDLL(t5a_probe_so)
    for name in ("probe_t5_dense", "probe_t5a_records"):
        getattr(lib, name)


def test_dense_coefficients_are_the_published_weights():
    """No GPU needed: R restates b_j(theta) (the expansion the records' c0..c3 are checked against), and sum_j b_j(1) k_j
    is the step's own b row (b_7 = 0)."""
    for j in range(7):
        for th in (0.25, 0.5, 0.9, 1.0):
            assert sum(R_EXACT[j][m] * Fraction(th) ** (m + 1) for m in range(4)) == b_exact(j, th)
        b = Fraction(A_TXT[6][j]) if j < 6 else Fraction(0)
        assert abs(float(sum(R_EXACT[j])) - float(b)) <= 1e-15


@pytest.fixture(scope="module")
def lv_clone_registered():
    return register_lv_clone()


@pytest.fixture(scope="module")
def probe(t5a_probe_so):
    lib = C.CDLL(t5a_probe_so)
    vp, i = C.c_void_p, C.c_int
    lib.probe_t5_dense.argtypes = [i, i, vp, vp, vp, i, C.c_longlong, i, vp, vp, vp, vp, vp]
    lib.probe_t5a_records.argtypes = [vp, vp, vp, vp, vp, vp, vp, vp, vp]
    return lib


def _check(rc):
    assert rc == 0, f"probe failed: cudaError {rc}"


# ------------------------------------------------------------------------------------------------------------------------
# T5Dense<D>::eval


def _knot_set(kind, m, rng):
    """knots of one member: kind 0 geometric, 1 dyadic, 2 with a one-ulp interval (an event step), 3 a single interval,
    4 forty-odd intervals of random lengths; m varies the count so that the lanes of a warp differ"""
    if kind == 0:
        kn = np.concatenate([[0.0], 1e-3 * 1.6 ** np.arange(4 + m % 13)])
    elif kind == 1:
        kn = np.arange(3 + m % 17) / 8.0 + 0.25 * (m % 3)
    elif kind == 2:
        kn = np.sort(rng.uniform(0.0, 2.0, 4 + m % 9))
        j = 1 + m % (len(kn) - 2)
        kn = np.insert(kn, j + 1, np.nextafter(kn[j], np.inf))
    elif kind == 3:
        kn = np.array([0.5, 0.5 + 1.5 * (1 + m % 5)])
    else:
        kn = np.concatenate([[0.0], np.cumsum(rng.uniform(0.01, 0.2, 40 + m % 11))])
    return np.unique(kn)


def _records(kn, D, rng):
    """member-major records [n + 1][8 D + 4] as the forward kernel writes them: (u, c0..c3, 0 x 3 D, t_n, h, 1/h, t_{n+1});
    the terminal record holds u and t only"""
    n = len(kn) - 1
    rec = np.zeros((n + 1, 8 * D + 4))
    rec[:, :D] = rng.standard_normal((n + 1, D))
    for k in range(n):
        rec[k, D:5 * D] = rng.standard_normal(4 * D) * 3.0
        h = kn[k + 1] - kn[k]
        rec[k, 8 * D:] = [kn[k], h, 1.0 / h, kn[k + 1]]
    rec[n, 8 * D], rec[n, 8 * D + 3] = kn[n], kn[n]
    return rec


def _walk(kn, rng, Q):
    """a query walk as the reverse solve makes it: downwards, several lookups per step (the stage times with continuity
    right, Gauss nodes left), every knot with both continuities and one ulp either side, jumps down over 1 to 5 intervals,
    upward moves (left then right at an event), and t0, T and points outside [t0, T]"""
    t0, T = kn[0], kn[-1]
    n = len(kn) - 1
    out = [(T, 1), (T, 0), (np.nextafter(T, np.inf), 1), (T + 1.0, 0)]
    t = T
    while len(out) < Q - 6 and t > t0:
        hs = -min(t - t0, (T - t0) * rng.uniform(0.002, 0.1))
        tn = t + hs if t + hs > t0 else t0
        out += [(t, 1), (t + 0.3 * hs, 1), (t + 0.5 * hs, 0), (tn, 1)]
        inside = kn[(kn >= tn) & (kn <= t)][::-1]
        out += [(k, 1) for k in inside]         # knot to knot downwards: the prefetched record of the interval below
        for k in inside:
            out += [(k, 1), (k, 0), (np.nextafter(k, np.inf), 1), (np.nextafter(k, -np.inf), 0), (np.nextafter(k, -np.inf), 1)]
        u = rng.uniform()
        if u < 0.08:                          # an event: the left limit, then the right one, a little above
            te = min(T, tn + (T - t0) * rng.uniform(0.0, 0.05))
            out += [(te, 0), (te, 1)]
        elif u < 0.16:                        # a jump down over 1 to 5 intervals
            iv = dense_interval(kn, n, tn, True)
            tn = max(t0, kn[max(0, iv - int(rng.integers(1, 6)))] + 0.5 * (kn[1] - kn[0]) * rng.uniform())
        t = tn
    out += [(t0, 1), (t0, 0), (np.nextafter(t0, -np.inf), 1), (t0 - 1.0, 0), (0.5 * (t0 + T), 1), (T, 1)]
    while len(out) < Q:
        out.append((rng.uniform(t0 - 0.1, T + 0.1), int(rng.integers(0, 2))))
    return out[:Q]


def dense_walk(kn, queries):
    """T5Dense's buffer state machine restated: -> (interval, buffer) after each query.  A lookup outside the held interval
    takes the prefetched record of the interval below if `holds()` accepts it there (the buffers swap), else the cursor
    search reloads the current buffer; either way the interval below the new one is prefetched into the other buffer."""
    n = len(kn) - 1

    def holds(iv, ta, tb, t, right):
        if right:
            return (iv == 0 or ta <= t) and (iv == n - 1 or tb > t)
        return (iv == 0 or ta < t) and (iv == n - 1 or tb >= t)

    cur, cb, civ, aiv, cta, ctb, out = n - 1, 0, -1, -1, 0.0, 0.0, []
    for t, right in queries:
        if not (civ >= 0 and holds(civ, cta, ctb, t, right)):
            got = False
            if aiv >= 0 and holds(aiv, kn[aiv], cta, t, right):
                cb, civ, ctb, cta, cur, got = cb ^ 1, aiv, cta, kn[aiv], aiv, True
            if not got:
                civ = cur = dense_interval(kn, n, t, right)
                cta, ctb = kn[civ], kn[civ + 1]
            aiv = civ - 1
        out.append((civ, cb))
    return out


def dense_eval_t5(rec, iv, t, D):
    """y of interval iv with the kernel's operations: h = t_{n+1} - t_n, theta = (t - t_n) * (1/h), g = h theta,
    y = fma(g, fma(th, fma(th, fma(th, c3, c2), c1), c0), u)"""
    r, r1 = rec[iv], rec[iv + 1]
    ta = r[8 * D]
    h = r1[8 * D] - ta
    th = 1.0 if h == 0.0 else (t - ta) * r[8 * D + 2]
    g = h * th
    return np.array([fma(g, fma(th, fma(th, fma(th, r[4 * D + j], r[3 * D + j]), r[2 * D + j]), r[D + j]), r[j]) for j in range(D)])


@pytest.mark.gpu
@pytest.mark.parametrize("D", [1, 2, 3])
def test_t5_dense_lookups(probe, D):
    rng = np.random.default_rng(70 + D)
    N, Q = 165, 160
    sets = [_knot_set(i % 5, i // 5, rng) for i in range(N)]
    nmax = max(len(s) - 1 for s in sets)
    stride, REC = nmax + 1, 8 * D + 4
    recs, knots = np.zeros((N, stride, REC)), np.zeros((N, stride))
    nk = np.array([len(s) - 1 for s in sets], dtype=np.int32)
    tq, rq = np.zeros((N, Q)), np.zeros((N, Q), dtype=np.int32)
    for i, kn in enumerate(sets):
        recs[i, :len(kn)] = _records(kn, D, rng)
        knots[i, :len(kn)] = kn
        for k, (t, r) in enumerate(_walk(kn, rng, Q)):
            tq[i, k], rq[i, k] = t, r
    assert len(set(nk[:32])) > 8 and nk.max() >= 40 and nk.min() == 1
    want_iv = np.array([[dense_interval(sets[i], nk[i], tq[i, k], bool(rq[i, k])) for k in range(Q)] for i in range(N)])
    walk = np.array([dense_walk(sets[i], [(tq[i, k], bool(rq[i, k])) for k in range(Q)]) for i in range(N)])
    assert np.array_equal(walk[:, :, 0], want_iv)          # the state machine lands where the scan does
    swaps = (np.diff(walk[:, :, 1], axis=1) != 0).sum()
    assert swaps > N                                        # the prefetch path is taken, not only the cursor search
    want_y = np.array([[dense_eval_t5(recs[i], want_iv[i, k], tq[i, k], D) for k in range(Q)] for i in range(N)])
    for block in (32, 64, 128):
        assert N % block
        y, iv, buf = np.zeros((N, Q, D)), np.zeros((N, Q), dtype=np.int32), np.zeros((N, Q), dtype=np.int32)
        _check(_dense_on_device(probe, D, block, recs, knots, nk, stride, N, Q, tq, rq, y, iv, buf))
        bad = np.argwhere(iv != want_iv)
        assert not len(bad), [(block, i, k, tq[i, k], rq[i, k], iv[i, k], want_iv[i, k]) for i, k in bad[:5]]
        bad = np.argwhere((y != want_y).any(axis=2))
        assert not len(bad), [(block, i, k, tq[i, k], rq[i, k], y[i, k], want_y[i, k]) for i, k in bad[:5]]
        bad = np.argwhere(buf != walk[:, :, 1])
        assert not len(bad), [(block, i, k, tq[i, k], rq[i, k], buf[i, k]) for i, k in bad[:5]]


def _dense_on_device(probe, D, block, recs, knots, nk, stride, N, Q, tq, rq, y, iv, buf):
    import torch
    dev = [torch.tensor(np.ascontiguousarray(a), device="cuda") for a in (recs, knots, nk, tq, rq)]
    yd, ivd = torch.zeros(y.shape, dtype=torch.float64, device="cuda"), torch.zeros(iv.shape, dtype=torch.int32, device="cuda")
    bd = torch.zeros(buf.shape, dtype=torch.int32, device="cuda")
    rc = probe.probe_t5_dense(D, block, dev[0].data_ptr(), dev[1].data_ptr(), dev[2].data_ptr(), stride, N, Q, dev[3].data_ptr(),
                              dev[4].data_ptr(), yd.data_ptr(), ivd.data_ptr(), bd.data_ptr())
    y[...], iv[...], buf[...] = yd.cpu().numpy(), ivd.cpu().numpy(), bd.cpu().numpy()
    return rc


# ------------------------------------------------------------------------------------------------------------------------
# the stored forward and reverse steps, the controller decisions


T40, T64 = None, None


def _tabs():
    global T40, T64
    if T40 is None:
        with mp.workdps(DPS):
            T40 = Tab(mp.mpf)
        T64 = Tab(float)
    return T40, T64


def t5_stages(tab, rhs, t, h, z):
    """the seven stages of one Tsit5 step from (t, z) and the end point z + h sum b k (number type of tab and rhs)"""
    L = len(z)
    k = [rhs(t, z)]
    for s in range(1, 7):
        zs = [z[c] + h * sum(tab.A[s][j] * k[j][c] for j in range(s)) for c in range(L)]
        k.append(rhs(fma(C64[s], float(h), t), zs))          # the stage time in fp64, as the kernels form it
    return k, zs


def t5_eest(tab, h, z, zn, k, abstol, reltol):
    """sqrt(mean((h sum_j btilde_j k_j / (abstol + reltol max(|z|, |zn|)))^2))"""
    e2 = 0
    for c in range(len(z)):
        e = h * sum(tab.BT[j] * k[j][c] for j in range(7))
        e2 += (e / (abstol + reltol * max(abs(z[c]), abs(zn[c])))) ** 2
    return (mp.sqrt if isinstance(e2, mp.mpf) else np.sqrt)(e2 / len(z))


def t5_eabs(tab, h, z, zn, k, abstol, reltol):
    """the estimate with every term taken by magnitude: eps times this bounds the rounding of the sum itself"""
    e2 = 0.0
    for c in range(len(z)):
        e = abs(h) * sum(abs(tab.BT[j] * k[j][c]) for j in range(7))
        e2 += (e / (abstol + reltol * max(abs(z[c]), abs(zn[c])))) ** 2
    return float(np.sqrt(e2 / len(z)))


def _jnorm(f, u, p):
    """infinity norm of df/du at u (fp64 complex steps)"""
    J = np.zeros((len(u), len(u)))
    for c in range(len(u)):
        uc = [complex(v) for v in u]
        uc[c] += 1e-60j
        J[:, c] = [complex(v).imag / 1e-60 for v in f(uc, [complex(float(v)) for v in p])]
    return np.abs(J).sum(axis=1).max()


OBS = {}          # largest observed error / bound of every check kind in this session (printed by the tests)


def _seen(kind, err, bound):
    OBS[kind] = max(OBS.get(kind, 0.0), float(err) / float(bound) if bound > 0 else (0.0 if err == 0 else np.inf))


def _ulp(x):
    return np.spacing(abs(float(x)))


class Controller:
    """the PI controller of both kernels, with the relative uncertainty rho of the proposed step that the fp64 rounding of
    the kernels' estimates leaves (see the module docstring)"""

    def __init__(self, h):
        self.h, self.qold, self.qold_rel, self.rho, self.habs = h, 1e-4, 0.0, 0.0, 0.0
        self.margin, self.rejects, self.decisions, self.closest = np.inf, 0, 0, None
        self.small = 0                    # accepted steps with EEst < 1e-4 (qold takes the floor 1e-4, not EEst)

    @staticmethod
    def _rounding(e, est):
        """relative fp64 rounding of the kernels' estimate e: 16 times the difference of an fp64 evaluation (est[0]) from the
        40-digit one, at least 16 eps times the magnitude sum (est[1])"""
        return max(16 * abs(est[0] - e) / e, 16 * EPS * est[1] / e, 64 * EPS) if e > 0 else 0.0

    def decide(self, e40, est, h):
        """accept or reject an attempt of step h (clipped); on a rejection the next attempt's h is set"""
        e = float(e40)
        e_rel = self._rounding(e, est) + 5 * (self.rho + self.habs / abs(h)) if e > 0 else 0.0
        m = abs(e40 - 1) / max(1e-6, 4 * e_rel * e)
        if m < self.margin:
            self.margin, self.closest = m, (e, e_rel)
        self.decisions += 1
        if e > 1.0:
            div = min(5.0, max(e, 1e-300) ** (7.0 / 50.0) / 0.9)
            self.rejects += 1
            self.h, self.habs, self.rho = h / div, self.habs / div, self.rho + 0.14 * e_rel
            return False
        return True

    def accept(self, e40, est, h_rec, h_unc, exact):
        """the accepted step as recorded (h_rec, within h_unc of the kernel's h; its estimate e40 recomputed at h_rec) -> the
        next proposal h_rec / q, and qold"""
        e = float(e40)
        e_rel = self._rounding(e, est) + 5 * h_unc / abs(h_rec) if e > 0 else 0.0
        q11 = max(e, 1e-300) ** (7.0 / 50.0)
        q = max(1.0 / 10.0, min(5.0, q11 / self.qold ** (2.0 / 25.0) / 0.9))
        self.h, self.rho, self.habs = h_rec / q, 0.14 * e_rel + 0.08 * self.qold_rel, (0.0 if exact else h_unc / q)
        self.qold, self.qold_rel = max(e, 1e-4), (e_rel if e > 1e-4 else 0.0)
        self.small += e < 1e-4

    def check_accepted(self, h_used, h_rec, t_next, what):
        tol = 4 * self.rho * abs(h_rec) + 4 * self.habs + 16 * _ulp(t_next)
        _seen("h replay", abs(h_used - h_rec), tol)
        assert abs(h_used - h_rec) <= tol, (what, h_used, h_rec, tol)


def _t5_problem(family, N, shared_p):
    """the Rosenbrock23 reference's problems; Robertson with mild rates (k = 0.4, 30, 10) that an explicit solver takes in
    a few hundred steps"""
    t0, T, saveat, u0, p = problem(family, N, shared_p)
    if family == "robertson":
        rng = np.random.default_rng(33)
        p = np.array([0.4, 30.0, 10.0])
        if not shared_p:
            p = p[:, None] * np.exp(0.05 * rng.standard_normal((3, N)))
    return t0, T, saveat, u0, p


def _member_p(p, shared_p, i):
    return list(p) if shared_p else list(p[:, i])


def _records_of(probe, eng, reverse=False):
    """(knots[N][maxs+1], records[N][maxs+1][8d+4], fn[N]) and, after a QuadratureAdjoint pass, (rrec, rend, rn)"""
    ms, rwp = C.c_int(), C.c_int()
    h = eng.handle._h
    _check(probe.probe_t5a_records(h, C.byref(ms), C.byref(rwp), None, None, None, None, None, None))
    N, d, M = eng.N, eng.d, ms.value
    ft, fr, fn = np.zeros((N, M + 1)), np.zeros((N, M + 1, 8 * d + 4)), np.zeros(N, dtype=np.int32)
    out = [ft, fr, fn]
    if reverse:
        out += [np.zeros((N, M, rwp.value)), np.zeros((N, M)), np.zeros(N, dtype=np.int32)]
    ptrs = [a.ctypes.data for a in out] + [None] * (6 - len(out))
    _check(probe.probe_t5a_records(h, C.byref(ms), C.byref(rwp), *ptrs))
    return out


def check_forward_member(f, p, kn, rec, n, t0, t1, dt0, abstol, reltol, fixed):
    """every stored record of one member, and every controller decision that led to it; -> the Controller"""
    tab40, tab64 = _tabs()
    D = (rec.shape[1] - 4) // 8
    assert kn[0] == t0 and kn[n] == t1 and n >= 1
    fin = rec[n]
    assert fin[8 * D] == t1 and fin[8 * D + 3] == t1 and fin[8 * D + 1] == 0 and fin[8 * D + 2] == 0 and not fin[D:8 * D].any()
    ctl = Controller(dt0 if dt0 > 0 else 1e-3 * (t1 - t0))
    p40 = [mp.mpf(float(v)) for v in p]
    rhs40, rhs64 = (lambda tt, x: f(x, p40)), (lambda tt, x: f(x, [float(v) for v in p]))
    t = t0
    for m in range(n):
        r = rec[m]
        u64, c, pad = r[:D], r[D:5 * D].reshape(4, D), r[5 * D:8 * D]
        ta, hr, ih, tb = r[8 * D:8 * D + 4]
        assert ta == kn[m] == t and tb == kn[m + 1] and hr == tb - ta and ih == 1.0 / hr and not pad.any(), (m, r[8 * D:])
        u40 = [mp.mpf(float(v)) for v in u64]
        # the controller: attempts until one is accepted
        while True:
            h = ctl.h
            last = False
            if t + h >= t1 or abs(t + h - t1) < 100 * 2.22e-16 * abs(t1):
                h, last = t1 - t, True
            if fixed:
                break
            k40, un40 = t5_stages(tab40, rhs40, t, h, u40)
            k64, un64 = t5_stages(tab64, rhs64, t, h, list(u64))
            est = (t5_eest(tab64, h, u64, un64, k64, abstol, reltol), t5_eabs(tab64, h, u64, un64, k64, abstol, reltol))
            if ctl.decide(t5_eest(tab40, h, u40, un40, k40, abstol, reltol), est, h):
                break
        if fixed:
            assert h == (t1 - t if last else dt0) and tb == (t1 if last else t + dt0), (m, t, h, tb)
        else:
            ctl.check_accepted(h, hr, tb, ("forward", m, t, last))
            assert (tb == t1) == last, (m, t, h, tb, last)
        # the record: stages in 40 digits from its own u_n, t_n and h.  The fp64 stages of the kernel carry the rounding of
        # their stage states, eps |u| passed on by the Jacobian: the bounds add 16 eps |J| |u| per stage
        k40, un40 = t5_stages(tab40, rhs40, ta, mp.mpf(hr), u40)
        ju = 16 * EPS * _jnorm(f, u64, p) * np.abs(u64).max()
        for mm in range(4):
            for j in range(D):
                terms = [tab40.R[s][mm] * k40[s][j] for s in range(7)]
                bound = 1e-14 * sum(abs(v) for v in terms) + ju * sum(abs(tab40.R[s][mm]) for s in range(7))
                _seen("c0..c3", abs(c[mm, j] - sum(terms)), bound)
                assert abs(c[mm, j] - sum(terms)) <= bound, (m, mm, j, c[mm, j], float(sum(terms)), float(bound))
        nxt = rec[m + 1][:D]
        for j in range(D):
            scale = abs(u40[j]) + abs(hr) * sum(abs(tab40.A[6][s]) * (abs(k40[s][j]) + ju / (16 * EPS)) for s in range(6))
            _seen("next u", abs(nxt[j] - un40[j]), 16 * EPS * scale)
            assert abs(nxt[j] - un40[j]) <= 16 * EPS * scale, (m, j, nxt[j], float(un40[j]), float(scale))
        if not fixed:           # the forward pass stores t_{n+1} - t_n: within an ulp of t_{n+1} of the kernel's h
            k64, un64 = t5_stages(tab64, rhs64, ta, hr, list(u64))
            est = (t5_eest(tab64, hr, u64, un64, k64, abstol, reltol), t5_eabs(tab64, hr, u64, un64, k64, abstol, reltol))
            ctl.accept(t5_eest(tab40, hr, u40, un40, k40, abstol, reltol), est, hr, _ulp(tb), False)
        t = tb
    assert t == t1
    return ctl


def _y40(rec, kn, n, t, D):
    """the forward solution at t in 40 digits from the (verified) records, right-continuous lookup"""
    iv = dense_interval(kn, n, t, True)
    r = rec[iv]
    h = mp.mpf(kn[iv + 1]) - mp.mpf(kn[iv])
    th = (mp.mpf(t) - mp.mpf(kn[iv])) / h
    return [r[j] + h * th * (r[D + j] + th * (r[2 * D + j] + th * (r[3 * D + j] + th * r[4 * D + j]))) for j in range(D)]


def check_reverse_member(f, p, kn, rec, n, rr, re, nr, saveat, t0, T, dt0, abstol, reltol, fixed, cost):
    """every stored reverse step of QuadratureAdjoint (lambda only, L = D) and every reverse controller decision"""
    tab40, tab64 = _tabs()
    D = (rec.shape[1] - 4) // 8
    p40, p64 = [mp.mpf(float(v)) for v in p], [float(v) for v in p]

    def rhs40(tt, x):
        return [-v for v in vjp_u(f, _y40(rec, kn, n, tt, D), p40, x)]

    def rhs64(tt, x):
        y = [complex(float(v)) for v in _y40(rec, kn, n, tt, D)]
        out = []
        for c in range(D):
            yc = list(y)
            yc[c] += 1e-60j
            out.append(-sum(x[r] * complex(v) for r, v in enumerate(f(yc, [complex(v) for v in p64]))).imag / 1e-60)
        return out

    cur = len(saveat) - 1
    z40 = [mp.mpf(0)] * D

    def jump_if_at(tt, z):
        nonlocal cur
        while cur >= 0 and abs(saveat[cur] - tt) <= EPS100 * max(abs(tt), 1.0):
            y = _y40(rec, kn, n, saveat[cur], D)
            z = [z[j] + cost[0] * y[j] + cost[1] for j in range(D)]
            cur -= 1
        return z

    z40 = jump_if_at(T, z40)
    ctl = Controller(-dt0 if dt0 > 0 else -1e-4 * (T - t0))
    t = T
    for m in range(nr):
        r = rr[m]
        tr, hr, zr, kr, ih = r[0], r[1], r[2:2 + D], r[2 + D:2 + 8 * D].reshape(7, D), r[2 + 8 * D]
        assert tr == t and ih == 1.0 / hr and re[m] == tr + hr, (m, tr, t, hr, re[m])
        zs = max(abs(v) for v in z40)
        _seen("next z", max(abs(zr[j] - z40[j]) for j in range(D)), 1e-13 * max(zs, 1e-300))
        assert all(abs(zr[j] - z40[j]) <= 1e-13 * max(zs, 1e-300) for j in range(D)), (m, zr, [float(v) for v in z40])
        zr40 = [mp.mpf(float(v)) for v in zr]
        while True:
            tstop = t0
            if cur >= 0 and t > saveat[cur] > tstop:
                tstop = saveat[cur]
            tn = tstop_snap(t + ctl.h, tstop)
            if tn < tstop:
                tn = tstop
            hs = tn - t
            if fixed:
                break
            k40, zn40 = t5_stages(tab40, rhs40, t, hs, zr40)
            k64, zn64 = t5_stages(tab64, rhs64, t, hs, list(zr))
            est = (t5_eest(tab64, hs, list(zr), zn64, k64, abstol, reltol), t5_eabs(tab64, hs, list(zr), zn64, k64, abstol, reltol))
            if ctl.decide(t5_eest(tab40, hs, zr40, zn40, k40, abstol, reltol), est, hs):
                break
        if fixed:
            assert hs == hr, (m, t, hs, hr)
        else:
            ctl.check_accepted(hs, hr, tr + hr, ("reverse", m, t))
        # the stored stages against 40 digits from the record's own z, t and h
        k40, zn40 = t5_stages(tab40, rhs40, tr, mp.mpf(hr), zr40)
        ks = max(abs(v) for s in k40 for v in s)
        bound = 1e-13 * ks + 64 * EPS * _jnorm(f, [float(v) for v in _y40(rec, kn, n, tr, D)], p) * float(max(abs(v) for v in zr40))
        err = max(abs(kr[s][j] - k40[s][j]) for s in range(7) for j in range(D))
        _seen("reverse stages", err, bound)
        assert err <= bound, (m, float(err), float(bound))
        if not fixed:           # the reverse pass stores its h
            k64, zn64 = t5_stages(tab64, rhs64, tr, hr, list(zr))
            est = (t5_eest(tab64, hr, list(zr), zn64, k64, abstol, reltol), t5_eabs(tab64, hr, list(zr), zn64, k64, abstol, reltol))
            ctl.accept(t5_eest(tab40, hr, zr40, zn40, k40, abstol, reltol), est, hr, 0.0, True)
        # the next step starts at the snapped end point tn; rend = t + h may differ from it by the rounding of t + h
        t = rr[m + 1][0] if m + 1 < nr else t0
        assert t == tn or abs(t - re[m]) <= _ulp(t), (m, t, tn, re[m])
        z40 = jump_if_at(t, zn40)
    assert t == t0 and cur < 0
    return ctl


FWD_RUNS = [  # family, shared p, tolerance, first step dt0 (> 0: a first step that the controller rejects)
    ("lv", True, 1e-6, 0.0), ("lv", False, 1e-10, 0.5),
    ("lorenz", False, 1e-6, 0.2), ("lorenz", True, 1e-9, 0.0),
    ("robertson", False, 1e-6, 3.0), ("robertson", True, 1e-10, 0.0),
    ("lv_clone", False, 1e-8, 0.5)]
FIXED_RUNS = [("lv", False, 0.02), ("lorenz", True, 0.005)]       # constant step, off-grid save times
N_FWD = 3


def _engine(family, sensealg, shared_p, tol, dt0, N, fixed=False, saveat=None, t=None):
    import scimlsensitivity_jl_b200 as b
    t0, T, sv, u0, p = _t5_problem(family, N, shared_p)
    saveat = sv if saveat is None else saveat
    eng = b.DeviceEnsemble(family, sensealg, "tsit5_fixed" if fixed else "tsit5_adaptive", N, saveat, (t0, T), dt0, shared_p=shared_p,
                           cost=b.AffineCost(1.0, -0.5), abstol=tol, reltol=tol, quad_abstol=1e-8, quad_reltol=1e-8, max_steps=4096)
    saved, status = eng.forward(u0, p)
    assert (np.asarray(status) == 0).all()
    return eng, (t0, T, saveat, u0, p)


@pytest.mark.gpu
def test_every_stored_forward_step_and_controller_decision(probe, lv_clone_registered):
    rejects = {}
    for family, shared_p, tol, dt0 in FWD_RUNS:
        f = FAMS[family][0]
        eng, (t0, T, saveat, u0, p) = _engine(family, "interpolating", shared_p, tol, dt0, N_FWD)
        kn, rec, fn = _records_of(probe, eng)
        eng.close()
        with mp.workdps(DPS):
            for i in range(N_FWD):
                ctl = check_forward_member(f, _member_p(p, shared_p, i), kn[i], rec[i], fn[i], t0, T, dt0, tol, tol, False)
                assert ctl.margin > 1.0, (family, i, ctl.margin, ctl.closest)
                rejects[family] = rejects.get(family, 0) + ctl.rejects
        print(f"forward {family} shared={shared_p} tol={tol:g} dt0={dt0}: steps {list(fn)}")
    print("rejected steps per family:", rejects, "observed error / bound:", OBS)
    assert all(v > 0 for v in rejects.values()), rejects


@pytest.mark.gpu
@pytest.mark.parametrize("family,shared_p,dt", FIXED_RUNS)
def test_constant_step_records(probe, family, shared_p, dt):
    f = FAMS[family][0]
    T = _t5_problem(family, 1, True)[1]
    saveat = np.array([0.0513, 0.1777, 0.31, 0.4421]) if family == "lorenz" else np.linspace(0.25, T, 8) + 0.003
    saveat[-1] = min(saveat[-1], T)
    eng, (t0, T, saveat, u0, p) = _engine(family, "interpolating", shared_p, 1e-6, dt, N_FWD, fixed=True, saveat=saveat)
    kn, rec, fn = _records_of(probe, eng)
    eng.close()
    with mp.workdps(DPS):
        for i in range(N_FWD):
            check_forward_member(f, _member_p(p, shared_p, i), kn[i], rec[i], fn[i], t0, T, dt, 1e-6, 1e-6, True)


@pytest.mark.gpu
def test_c1_ensemble_forward_records(probe):
    """the C1 bench configuration at its full size: 65 536 members, LV, shared p, tolerance 1e-8, T = 10, 101 save
    times; 64 members checked, among them the first and the last block's"""
    import scimlsensitivity_jl_b200 as b
    N, T = 65536, 10.0
    rng = np.random.default_rng(0)
    saveat = np.linspace(0.0, T, 101)
    u0 = np.exp(0.2 * rng.standard_normal((2, N)))
    p = np.array([1.5, 1.0, 3.0, 1.0])
    eng = b.DeviceEnsemble("lv", "interpolating", "tsit5_adaptive", N, saveat, (0.0, T), 0.0, cost=b.AffineCost(0.0, 1.0),
                           max_steps=512, abstol=1e-8, reltol=1e-8)
    _, status = eng.forward(u0, p)
    assert (status == 0).all()
    kn, rec, fn = _records_of(probe, eng)
    eng.close()
    pick = sorted(set(list(range(8)) + list(range(N - 8, N)) + list(rng.choice(N, 48, replace=False))))[:64]
    with mp.workdps(DPS):
        for i in pick:
            ctl = check_forward_member(f_lv, p, kn[i], rec[i], fn[i], 0.0, T, 0.0, 1e-8, 1e-8, False)
            assert ctl.margin > 1.0, (i, ctl.margin, ctl.closest)
    print("C1 members", len(pick), "observed error / bound:", OBS)


REV_RUNS = [("lv", False, 1e-6, 0.5, False), ("lorenz", True, 1e-8, 0.0, False), ("robertson", False, 1e-6, 3.0, False),
            ("lv", True, 1e-6, 0.02, True)]
N_REV = 2


@pytest.mark.gpu
@pytest.mark.parametrize("family,shared_p,tol,dt0,fixed", REV_RUNS)
def test_every_quadrature_reverse_step(probe, family, shared_p, tol, dt0, fixed):
    f = FAMS[family][0]
    saveat = None
    if fixed:
        saveat = np.linspace(0.25, 2.0, 8) + 0.003
        saveat[-1] = 2.0
    eng, (t0, T, saveat, u0, p) = _engine(family, "quadrature", shared_p, tol, dt0, N_REV, fixed=fixed, saveat=saveat)
    eng.reverse()
    kn, rec, fn, rr, re, rn = _records_of(probe, eng, reverse=True)
    eng.close()
    rejects = small = 0
    with mp.workdps(DPS):
        for i in range(N_REV):
            pi = _member_p(p, shared_p, i)
            check_forward_member(f, pi, kn[i], rec[i], fn[i], t0, T, dt0, tol, tol, fixed)
            ctl = check_reverse_member(f, pi, kn[i], rec[i], fn[i], rr[i], re[i], rn[i], list(saveat), t0, T, dt0, tol, tol, fixed, (1.0, -0.5))
            assert fixed or ctl.margin > 1.0, (i, ctl.margin, ctl.closest)
            rejects += ctl.rejects
            small += ctl.small
    print(f"reverse {family} shared={shared_p} tol={tol:g} dt0={dt0} fixed={fixed}: steps {list(rn)}, rejected {rejects}, "
          f"accepted with EEst < 1e-4: {small}; observed error / bound: {OBS}")
    if not fixed:     # steps accepted far below EEst = 1e-4 (the first one, those clipped at save times): qold takes its floor
        assert small > 0
    if dt0 > 0 and not fixed:
        assert rejects > 0
