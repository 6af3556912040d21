"""The fixed-step Tsit5 kernels (csrc/ode_tsit5.cuh) step by step, through tests/csrc/fixed_probe.cu: the production code
called unchanged, the forward checkpoints and QuadratureAdjoint's dense reverse solution read back from a handle.

* Every forward checkpoint (LV, Lorenz, Robertson with mild rates; shared and per-member p; fp64 and fp32; the interval
  checkpoint layout C = 3, S = 20; preset-time events that scale, shift and change parameters; 64 sampled members of C2
  at its full size, N = 65 536 and S = 1000): u_{n+1} against one Tsit5 step taken in extended precision (np.longdouble,
  eps <= 1.1e-19) from the device's own u_n, then the event affect where one fires.  Every step starts from the device's
  state, so nothing propagates and the bound is a few ulps:
      |u_{n+1} - U| <= eps (8 (|u_n| + sum_j |h b_j| |k_j|) + sum_{j<6} |h b_j| (8 F_j + |J(z_j)| Z_j)),
      Z_j = 8 eps (|u_n| + sum_{i<j} |h a_ji| |k_i|)
  where F_j is the sum of the magnitudes of the terms of f at stage state z_j (the rounding of one RHS evaluation),
  Z_j bounds the rounding of stage state z_j (its FMA chain and the one- or two-ulp rounding of the tables hA = h A)
  and |J| passes it to k_j; the first term is the final sum u_n + sum h b_j k_j.  Under interval checkpointing the
  C steps between stored rows compound: the bound of each is carried by exp(h ||J||) into the next.  Each fp64 run
  also shows that a relative change of 1e-10 in TSIT5_A[3][0] moves some u_{n+1} by more than 100 bounds.
* Every row QuadratureAdjoint's reverse pass stores (lambda(t_{n+1}) after the jump, ka'[0..6]): with u_n and u_{n+1}
  from the checkpoints, the forward stages recomputed from u_n and the exact dense output y_s = y(t_{n+1} - c_s h)
  (published b_j(theta)), ls_s = lambda + sum_j hA[s][j] ka_j, each ka_s against (df/du)'(y_s) ls_s (plus the
  continuous cost), the next row's lambda against ls_6 plus the loss jump at t_n, the first row's ka[0] against the
  jump at T, and du0 against the last step's ls_6 plus the jump at t0 (absent under no_start).  This pins the
  Hermite dense output with c4 from du (hC4u), the stage-time order, the jumps and no_start, step by step.  The bound
  is eps times the magnitudes of the terms, plus the dense output's own rounding: the device forms y from du = u_{n+1}
  - u_n, whose difference from the extended-precision step the Hermite weights (<= 1 + 15/16) pass on.

Observed on an H100 80GB HBM3 (700 W power limit), largest error as a share of its bound: forward checkpoints 0.21
(Robertson; LV 0.08, Lorenz 0.08, fp32 0.03, interval checkpoints 0.011, events 0.08, C2 at full size 0.10); reverse
stages ka_0..ka_6 0.13, next lambda 0.23, du0 0.18.  The 1e-10 change of TSIT5_A[3][0] moves u_{n+1} by 470 to 1250
bounds.  Together with tests/test_gpu_fixed_reference.py the module took 96 s of host time there.
"""
import ctypes as C
import os
import subprocess
from fractions import Fraction

import numpy as np
import pytest

import mpmath as mp

from scimlsensitivity_jl_b200 import _lib
from ros23_restatement import A_TXT, C_TXT, b_exact, f_lorenz, f_lv, f_robertson, fma

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
CSRC = os.path.join(ROOT, "scimlsensitivity.jl_b200", "csrc")
PROBE = os.path.join(ROOT, "tests", "csrc", "fixed_probe.cu")
LD = np.longdouble
EPS64, EPS32 = 2.220446049250313e-16, 1.1920928955078125e-07


def f_lv_abs(u, p):
    return [abs(p[0] * u[0]) + abs(p[1] * u[0] * u[1]), abs(p[2] * u[1]) + abs(p[3] * u[0] * u[1])]


def f_lorenz_abs(u, p):
    return [abs(p[0]) * (abs(u[1]) + abs(u[0])), abs(u[0]) * (abs(p[1]) + abs(u[2])) + abs(u[1]), abs(u[0] * u[1]) + abs(p[2] * u[2])]


def f_robertson_abs(y, k):
    return [abs(k[0] * y[0]) + abs(k[2] * y[1] * y[2]), abs(k[0] * y[0]) + abs(k[1] * y[1] * y[1]) + abs(k[2] * y[1] * y[2]), abs(k[1] * y[1] * y[1])]


# family: (f, magnitude of f's terms, d, P)
FAMS = {"lv": (f_lv, f_lv_abs, 2, 4), "lorenz": (f_lorenz, f_lorenz_abs, 3, 3), "robertson": (f_robertson, f_robertson_abs, 3, 3)}


def _ld(fr):
    """a Fraction (or decimal string) as a long double, to within its rounding"""
    fr = Fraction(fr)
    with mp.workdps(30):
        return LD(mp.nstr(mp.mpf(fr.numerator) / fr.denominator, 25))


A_LD = [[_ld(v) for v in row] for row in A_TXT]
C_F = [Fraction(c) for c in C_TXT]


def b_ld(th):
    """b_j(theta), j = 0..6, in long double from the published factored form"""
    return [_ld(b_exact(j, Fraction(th))) for j in range(7)]


@pytest.fixture(scope="session")
def fixed_probe_so(tmp_path_factory):
    """fixed_probe.cu built with the library's nvcc flags, once per session, outside the source tree."""
    so = str(tmp_path_factory.mktemp("fixed_probe") / "libfixed_probe.so")
    cmd = [_lib.nvcc_path(), "-gencode", "arch=compute_90a,code=sm_90a", "-O3", "-std=c++17", "-I", CSRC,
           "-Xcompiler", "-fPIC", "-shared", PROBE, "-o", so]
    res = subprocess.run(cmd, capture_output=True, text=True)
    assert res.returncode == 0, res.stdout[-3000:] + res.stderr[-3000:]
    return so


def test_fixed_probe_compiles_for_sm90a(fixed_probe_so):
    """No GPU needed: a header change that breaks the probe fails here."""
    assert C.CDLL(fixed_probe_so).probe_fixed_buffers
    assert np.finfo(LD).eps <= 1.1e-19        # the step-level restatement below runs in x87 extended precision


@pytest.fixture(scope="module")
def probe(fixed_probe_so):
    lib = C.CDLL(fixed_probe_so)
    vp, ip = C.c_void_p, C.POINTER(C.c_int)
    lib.probe_fixed_buffers.argtypes = [vp, ip, ip, ip, C.POINTER(C.c_longlong), ip, vp, vp]
    return lib


def buffers_of(probe, eng, reverse=False):
    """-> (S, C, ckpt[rows][d][N], adj[S][8][d][N] or None), the pad columns dropped"""
    S, rows, ck, es = C.c_int(), C.c_int(), C.c_int(), C.c_int()
    npad = C.c_longlong()
    h = eng.handle._h
    args = (C.byref(S), C.byref(rows), C.byref(ck), C.byref(npad), C.byref(es))
    assert probe.probe_fixed_buffers(h, *args, None, None) == 0
    dt = np.float64 if es.value == 8 else np.float32
    ckpt = np.zeros((rows.value, eng.d, npad.value), dtype=dt)
    adj = np.zeros((S.value, 8, eng.d, npad.value), dtype=dt) if reverse else None
    rc = probe.probe_fixed_buffers(h, *args, ckpt.ctypes.data, None if adj is None else adj.ctypes.data)
    assert rc == 0, f"probe failed: cudaError {rc}"
    return S.value, ck.value, ckpt[:, :, :eng.N], None if adj is None else adj[..., :eng.N]


OBS = {}          # largest observed error / bound of every check kind in this session (printed by the tests)


def _seen(kind, err, bound):
    r = np.max(np.asarray(err, dtype=np.float64) / np.asarray(bound, dtype=np.float64))
    OBS[kind] = max(OBS.get(kind, 0.0), float(r))


# ------------------------------------------------------------------------------------------------------------------------
# vectorised helpers: states are lists of D arrays over the members


def jac_abs_times(f, y, p, v):
    """|df/du (y)| v, the Jacobian by complex steps in fp64 (only magnitudes are needed)"""
    D = len(y)
    yc = [np.asarray(x, dtype=np.float64).astype(np.complex128) for x in y]
    pc = [np.asarray(q, dtype=np.float64).astype(np.complex128) for q in p]
    out = [np.zeros_like(yc[0].real) for _ in range(D)]
    for c in range(D):
        yy = list(yc)
        yy[c] = yy[c] + 1e-30j
        col = [np.abs(np.asarray(r).imag / 1e-30) for r in f(yy, pc)]
        for r in range(D):
            out[r] = out[r] + col[r] * np.asarray(v[c], dtype=np.float64)
    return out


def jac_norm(f, y, p):
    """||df/du (y)||_inf per member"""
    ones = [np.ones_like(np.asarray(y[0], dtype=np.float64)) for _ in y]
    return np.max(np.array(jac_abs_times(f, y, p, ones)), axis=0)


def vjp_u_ld(f, y, p, l):
    """(df/du)' l in long double, by complex steps (np.clongdouble)"""
    D = len(y)
    yc = [np.asarray(x, dtype=LD).astype(np.clongdouble) for x in y]
    pc = [np.asarray(q, dtype=LD).astype(np.clongdouble) for q in p]
    d = LD("1e-30")
    out = []
    for c in range(D):
        yy = list(yc)
        yy[c] = yy[c] + np.clongdouble(1j) * d
        out.append(sum(np.asarray(l[r], dtype=LD) * np.asarray(v).imag for r, v in enumerate(f(yy, pc))) / d)
    return out


def step_ld(f, u, p, h, A=A_LD):
    """one Tsit5 step in long double: (u_{n+1}, stages k[0..5], stage states z[0..5])"""
    D = len(u)
    k, z = [f(u, p)], [u]
    for s in range(1, 7):
        zs = [u[c] + h * sum(A[s][j] * k[j][c] for j in range(s)) for c in range(D)]
        if s < 6:
            z.append(zs)
            k.append(f(zs, p))
    return zs, k, z


def step_bound(f, fabs, u, p, h, k, z, eps):
    """the bound of the module docstring, per component"""
    D = len(u)
    hb = [abs(float(h) * float(A_LD[6][j])) for j in range(6)]
    au = [np.abs(np.asarray(x, dtype=np.float64)) for x in u]
    ak = [[np.abs(np.asarray(x, dtype=np.float64)) for x in kj] for kj in k]
    pa = [np.asarray(q, dtype=np.float64) for q in p]
    tot = [8 * (au[c] + sum(hb[j] * ak[j][c] for j in range(6))) for c in range(D)]
    for j in range(6):
        Zj = [8 * eps * (au[c] + sum(abs(float(h) * float(A_LD[j][i])) * ak[i][c] for i in range(j))) for c in range(D)]
        Fj = fabs([np.asarray(x, dtype=np.float64) for x in z[j]], pa)
        JZ = jac_abs_times(f, z[j], pa, Zj)
        for c in range(D):
            tot[c] = tot[c] + hb[j] * (8 * Fj[c] + JZ[c] / eps)
    return [eps * t for t in tot]


def params_after(p0, evs, upto, kind):
    """the parameters in force after the events at grid points <= upto, as the kernels form them (one FMA per event
    and parameter in the kernel's real type); p0: [P][M] in that type"""
    p = [np.array(q, dtype=np.float64) for q in p0]
    for n in sorted(evs):
        if n > upto:
            break
        _, _, ps, pc = evs[n]
        if ps is None:
            continue
        for q in range(len(p)):
            if kind == "f64":
                p[q] = np.array([fma(ps[q], v, pc[q]) for v in p[q]])
            else:
                p[q] = np.array([np.float32(Fraction(float(np.float32(ps[q]))) * Fraction(float(v)) + Fraction(float(np.float32(pc[q]))))
                                 for v in p[q]], dtype=np.float64)
    return p


def check_checkpoints(fam, ckpt, S, Cev, h, p_of, evs, eps, tag, sensitivity=True):
    """every stored forward checkpoint of the members in ckpt[rows][D][M] (values in the kernel's real type);
    p_of(n): the parameters of step n ([P][M] float64 values in the kernel's type); evs: {n: (s, c, ps, pc)}"""
    f, fabs, D, P = FAMS[fam]
    hL = LD(h)
    worst, moved = 0.0, 0.0
    rows = ckpt.shape[0]
    if Cev == 1:
        segs = [(n, n + 1, 1) for n in range(S)]
    else:
        nm = (S + Cev - 1) // Cev
        assert rows == nm + 1
        segs = [(m, m + 1, min(Cev, S - m * Cev)) for m in range(nm)]
    for r0, r1, steps in segs:
        n0 = r0 * Cev
        u = [ckpt[r0, c].astype(LD) for c in range(D)]
        carried = np.zeros(ckpt.shape[2])
        for q in range(steps):
            n = n0 + q
            p = [np.asarray(v, dtype=LD) for v in p_of(n)]
            un, k, z = step_ld(f, u, p, hL)
            b = step_bound(f, fabs, u, p_of(n), h, k, z, eps)
            grow = np.exp(h * jac_norm(f, u, p_of(n))) * 1.5
            bound = [carried * grow + bc for bc in b]
            if sensitivity and Cev == 1 and eps == EPS64:
                Am = [list(r) for r in A_LD]
                Am[3][0] = Am[3][0] * (1 + LD("1e-10"))
                um, _, _ = step_ld(f, u, p, hL, Am)
                moved = max(moved, float(np.max(np.array([np.abs(np.asarray(um[c] - un[c], dtype=np.float64)) / bound[c] for c in range(D)]))))
            if n + 1 in evs and n + 1 < S:
                s, cc, _, _ = evs[n + 1]
                un = [LD(s[c]) * un[c] + LD(cc[c]) for c in range(D)]
                bound = [abs(s[c]) * bound[c] + 4 * eps * (np.abs(np.asarray(un[c], dtype=np.float64)) + abs(cc[c])) for c in range(D)]
            u = un
            carried = np.max(np.array(bound), axis=0)
        for c in range(D):
            err = np.abs(ckpt[r1, c].astype(LD) - u[c]).astype(np.float64)
            _seen(f"forward {tag}", err, bound[c])
            bad = np.argwhere(err > bound[c])
            assert not len(bad), (tag, r1, c, [(int(i), err[i], bound[c][i]) for i in bad[:4, 0]])
            worst = max(worst, float(np.max(err / bound[c])))
    if sensitivity and Cev == 1 and eps == EPS64:
        OBS[f"TSIT5_A[3][0] * (1 + 1e-10) / bound, {tag}"] = moved
        assert moved > 100, (tag, moved)
    return worst


# ------------------------------------------------------------------------------------------------------------------------
# forward runs


def t5_problem(family, N, shared_p):
    """LV, Lorenz (T = 0.5) and Robertson with mild rates (k = 0.4, 30, 10) over T = 2"""
    rng = np.random.default_rng({"lv": 1, "lorenz": 2, "robertson": 3}[family])
    if family == "lv":
        T, u0, p = 2.0, np.exp(0.1 * rng.standard_normal((2, N))), np.array([1.5, 1.0, 3.0, 1.0])
    elif family == "lorenz":
        T, u0, p = 0.5, np.array([1.0, 0.0, 0.0])[:, None] + 0.1 * rng.standard_normal((3, N)), np.array([10.0, 28.0, 8.0 / 3.0])
    else:
        T, u0, p = 2.0, np.repeat(np.array([[1.0], [0.0], [0.0]]), N, 1) + 0.01 * np.abs(rng.standard_normal((3, N))), np.array([0.4, 30.0, 10.0])
    if not shared_p:
        p = p[:, None] * np.exp(0.05 * rng.standard_normal((len(p), N)))
    return T, u0, p


def member_params(p, shared_p, N, dtype):
    """[P][N] float64 arrays holding the values the kernel reads"""
    cast = (lambda a: np.asarray(a, dtype=np.float32).astype(np.float64)) if dtype == "f32" else (lambda a: np.asarray(a, dtype=np.float64))
    return [cast(np.full(N, q) if shared_p else p[i]) for i, q in enumerate(p if shared_p else range(len(p)))]


FWD_RUNS = [  # family, shared p, dt, dtype, checkpoint_every
    ("lv", True, 0.1, "f64", 1), ("lv", False, 0.05, "f64", 1), ("lorenz", True, 0.01, "f64", 1), ("lorenz", False, 0.025, "f64", 1),
    ("robertson", True, 0.05, "f64", 1), ("robertson", False, 0.02, "f64", 1),
    ("lv", False, 0.1, "f32", 1), ("lorenz", True, 0.025, "f32", 1),
    ("lv", True, 0.1, "f64", 3), ("lorenz", False, 0.025, "f64", 3)]
N_FWD = 70


@pytest.mark.gpu
@pytest.mark.parametrize("family,shared_p,dt,dtype,C", FWD_RUNS)
def test_every_forward_checkpoint(probe, family, shared_p, dt, dtype, C):
    import scimlsensitivity_jl_b200 as b
    T, u0, p = t5_problem(family, N_FWD, shared_p)
    if C > 1:
        T = 20 * dt                                        # S = 20, not a multiple of C = 3
    eng = b.DeviceEnsemble(family, "interpolating" if C == 1 else "gauss", "tsit5_fixed", N_FWD, [T], (0.0, T), dt, shared_p=shared_p,
                           cost=b.AffineCost(1.0, 0.0), dtype=dtype, checkpoint_every=C, block_threads=32)
    _, status = eng.forward(u0, p)
    assert (np.asarray(status) == 0).all()
    S, Cs, ckpt, _ = buffers_of(probe, eng)
    eng.close()
    assert Cs == C and S == int(round(T / dt))
    pm = member_params(p, shared_p, N_FWD, dtype)
    assert np.array_equal(ckpt[0], np.asarray(u0, dtype=ckpt.dtype))
    check_checkpoints(family, ckpt, S, C, dt, lambda n: pm, {}, EPS64 if dtype == "f64" else EPS32, f"{family} {dtype} C={C}")
    print(f"forward {family} shared={shared_p} dt={dt} {dtype} C={C}: observed error / bound {OBS}")


EV_TIMES = [0.5, 1.0, 1.5]


def lv_events(pchange):
    """LV on [0, 2], dt = 0.05: events that scale, shift and (pchange) change parameters"""
    s = np.array([[1.2, 0.9], [1.0, 1.1], [0.8, 1.0]])
    c = np.array([[0.1, 0.0], [-0.05, 0.2], [0.0, 0.0]])
    ps = np.array([[1.1, 1.0, 0.95, 1.0], [1.0, 1.05, 1.0, 0.9], [0.9, 1.0, 1.0, 1.1]]) if pchange else None
    pc = np.array([[0.0, 0.1, 0.0, -0.05], [0.02, 0.0, 0.1, 0.0], [0.0, -0.1, 0.0, 0.0]]) if pchange else None
    return s, c, ps, pc


@pytest.mark.gpu
@pytest.mark.parametrize("shared_p,pchange", [(True, False), (False, True), (True, True)])
def test_every_forward_checkpoint_with_events(probe, shared_p, pchange):
    """preset-time events on the dt grid: checkpoints hold the post-event state, later steps run on the new parameters"""
    import scimlsensitivity_jl_b200 as b
    dt, N = 0.05, 40
    T, u0, p = t5_problem("lv", N, shared_p)
    s, c, ps, pc = lv_events(pchange)
    eng = b.DeviceEnsemble("lv", "interpolating", "tsit5_fixed", N, [T], (0.0, T), dt, shared_p=shared_p, cost=b.AffineCost(1.0, 0.0))
    eng.set_events(EV_TIMES, s, c, ps, pc)
    _, status = eng.forward(u0, p)
    assert (np.asarray(status) == 0).all()
    S, _, ckpt, _ = buffers_of(probe, eng)
    eng.close()
    evs = {int(round(t / dt)): (s[e], c[e], None if ps is None else ps[e], None if pc is None else pc[e]) for e, t in enumerate(EV_TIMES)}
    p0 = member_params(p, shared_p, N, "f64")
    check_checkpoints("lv", ckpt, S, 1, dt, lambda n: params_after(p0, evs, n, "f64"), evs, EPS64, f"lv events pchange={pchange}")


@pytest.mark.gpu
def test_c2_forward_checkpoints_full_size(probe):
    """C2 at its full size (Lorenz, N = 65 536, dt = 0.01, S = 1000, shared p): 64 members, among them the first and the
    last block's, every checkpoint"""
    import scimlsensitivity_jl_b200 as b
    import bench
    W = bench.WORKLOAD
    N, T, dt = W["members_per_gpu"], W["T"], W["dt"]
    u0, p = bench.make_inputs(N)
    saveat = np.linspace(0.0, T, W["nsave"])
    eng = b.DeviceEnsemble("lorenz", "gauss", "tsit5_fixed", N, saveat, (0.0, T), dt, cost=b.AffineCost(*W["cost"]))
    _, status = eng.forward(u0, p)
    assert (np.asarray(status) == 0).all()
    S, _, ckpt, _ = buffers_of(probe, eng)
    eng.close()
    rng = np.random.default_rng(5)
    pick = np.array(sorted(set(list(range(8)) + list(range(N - 8, N)) + list(rng.choice(N, 48, replace=False))))[:64])
    sub = np.ascontiguousarray(ckpt[:, :, pick])
    del ckpt
    pm = member_params(p, True, len(pick), "f64")
    check_checkpoints("lorenz", sub, S, 1, dt, lambda n: pm, {}, EPS64, "C2 full size")
    print(f"C2 members {len(pick)}, steps {S}: observed error / bound {OBS}")


# ------------------------------------------------------------------------------------------------------------------------
# QuadratureAdjoint's reverse rows


THETA_S = [1 - C_F[s] for s in range(7)]          # adjoint stage s at y(t_{n+1} - c_s h)
BS = [b_ld(THETA_S[s]) for s in range(5)]


def vjp_abs(fabs, y, p, l):
    """sum of the magnitudes of the terms of (df/du)' l: the complex-step VJP of the magnitude function"""
    yy = [np.abs(np.asarray(x, dtype=np.float64)) for x in y]
    ll = [np.abs(np.asarray(x, dtype=np.float64)) for x in l]
    pp = [np.abs(np.asarray(q, dtype=np.float64)) for q in p]
    D = len(y)
    out = []
    for c in range(D):
        yc = [x.astype(np.complex128) for x in yy]
        yc[c] = yc[c] + 1e-30j
        out.append(sum(ll[r] * np.asarray(v).imag / 1e-30 for r, v in enumerate(fabs_c(fabs, yc, pp))))
    return out


def fabs_c(fabs, y, p):
    """the magnitude function at complex arguments (abs() would drop the imaginary part): magnitudes are polynomials with
    positive coefficients, so restate them without abs at the non-negative real point"""
    return {f_lv_abs: lambda u, q: [q[0] * u[0] + q[1] * u[0] * u[1], q[2] * u[1] + q[3] * u[0] * u[1]],
            f_lorenz_abs: lambda u, q: [q[0] * (u[1] + u[0]), u[0] * (q[1] + u[2]) + u[1], u[0] * u[1] + q[2] * u[2]],
            f_robertson_abs: lambda u, q: [q[0] * u[0] + q[2] * u[1] * u[2], q[0] * u[0] + q[1] * u[1] * u[1] + q[2] * u[1] * u[2], q[1] * u[1] * u[1]]}[fabs](y, p)


def check_quad_rows(fam, ckpt, adj, du0, S, h, pm, jump_of, cont, no_start, tag):
    """every stored reverse row; jump_of(n, u_n) -> the loss jump at grid point n (list of D arrays) or None"""
    f, fabs, D, P = FAMS[fam]
    hL = LD(h)
    p = [np.asarray(v, dtype=LD) for v in pm]
    eps = EPS64
    cA, cB = cont if cont else (0.0, 0.0)

    def add_cont(y, ka):
        return [ka[c] + LD(cA) * y[c] + LD(cB) for c in range(D)] if cont else ka

    lam_prev = None
    for n in range(S - 1, -1, -1):
        un = [ckpt[n, c].astype(LD) for c in range(D)]
        u1 = [ckpt[n + 1, c].astype(LD) for c in range(D)]
        lam = [adj[n, 0, c].astype(LD) for c in range(D)]
        ka = [[adj[n, 1 + s, c].astype(LD) for c in range(D)] for s in range(7)]
        # the forward step, its exact dense output and the device's Hermite form's extra rounding
        u1x, k, z = step_ld(f, un, p, hL)
        k.append(f(u1, p))                                  # k7 = f(u_{n+1}) at the checkpoint
        du_err = [np.abs(np.asarray(u1[c] - u1x[c], dtype=np.float64)) for c in range(D)]
        ys = [u1]
        yerr = [[np.zeros_like(du_err[0]) for _ in range(D)]]
        for s in range(1, 5):
            w = BS[s]
            # y from the device's u_{n+1}: u_n + sum_j h b_j(theta) k_j, with the (H01 + theta^2 (1-theta)^2 w_du) du
            # weight carrying the device's du in place of h sum b k
            th = float(THETA_S[s])
            hw = 3 * th ** 2 - 2 * th ** 3 + th ** 2 * (1 - th) ** 2 * 15.1
            y = [un[c] + hL * sum(w[j] * k[j][c] for j in range(7)) for c in range(D)]
            mag = [np.abs(np.asarray(un[c], dtype=np.float64)) + sum(abs(float(h) * float(w[j])) * np.abs(np.asarray(k[j][c], dtype=np.float64)) for j in range(7))
                   + float(h) * 47.4 * th ** 2 * (1 - th) ** 2 * sum(np.abs(np.asarray(k[j][c], dtype=np.float64)) for j in range(7)) for c in range(D)]
            ys.append(y)
            yerr.append([hw * du_err[c] + 16 * eps * mag[c] for c in range(D)])
        ys += [un, un]
        yerr += [[np.zeros_like(du_err[0]) for _ in range(D)]] * 2
        for s in range(7):
            ls = [lam[c] + hL * sum(A_LD[s][j] * ka[j][c] for j in range(s)) for c in range(D)] if s else lam
            lmag = [np.abs(np.asarray(lam[c], dtype=np.float64)) + sum(abs(float(h) * float(A_LD[s][j])) * np.abs(np.asarray(ka[j][c], dtype=np.float64)) for j in range(s))
                    for c in range(D)]
            want = add_cont(ys[s], vjp_u_ld(f, ys[s], p, ls))
            lerr = [8 * eps * lmag[c] for c in range(D)]
            # rounding of the VJP's own terms, the stage lambda's rounding through J', and the dense output's through
            # the second derivative (the magnitude VJP at y + yerr against y)
            g = vjp_abs(fabs, ys[s], pm, ls)
            jl = jac_abs_times(f, ys[s], pm, [np.ones_like(x) for x in lerr])
            ytop = [np.abs(np.asarray(ys[s][c], dtype=np.float64)) + yerr[s][c] for c in range(D)]
            g2 = vjp_abs(fabs, ytop, pm, ls)
            bound = [8 * eps * (g[c] + (abs(cA) * np.abs(np.asarray(ys[s][c], dtype=np.float64)) + abs(cB) if cont else 0))
                     + (g2[c] - g[c]) + abs(cA) * yerr[s][c] + np.max(np.array(lerr), axis=0) * jl[c] + 1e-300 for c in range(D)]
            for c in range(D):
                err = np.abs(np.asarray(ka[s][c] - want[c], dtype=np.float64))
                _seen(f"reverse ka_{s}", err, bound[c])
                bad = np.argwhere(err > bound[c])
                assert not len(bad), (tag, n, s, c, [(int(i), err[i], bound[c][i]) for i in bad[:4, 0]])
        # lambda(t_n): ls_6 plus the jump at t_n -> the next row, or du0
        l6 = [lam[c] + hL * sum(A_LD[6][j] * ka[j][c] for j in range(6)) for c in range(D)]
        l6mag = [np.abs(np.asarray(lam[c], dtype=np.float64)) + sum(abs(float(h) * float(A_LD[6][j])) * np.abs(np.asarray(ka[j][c], dtype=np.float64)) for j in range(6))
                 for c in range(D)]
        jmp = None if (no_start and n == 0) else jump_of(n, un)
        if jmp is not None:
            l6 = [l6[c] + LD(1) * jmp[c] for c in range(D)]
            l6mag = [l6mag[c] + np.abs(np.asarray(jmp[c], dtype=np.float64)) for c in range(D)]
        got = [adj[n - 1, 0, c] for c in range(D)] if n > 0 else [du0[c] for c in range(D)]
        for c in range(D):
            err = np.abs(np.asarray(got[c].astype(LD) - l6[c], dtype=np.float64))
            bnd = 8 * eps * l6mag[c] + 1e-300
            _seen("reverse next lambda" if n else "du0", err, bnd)
            assert (err <= bnd).all(), (tag, n, c, float(np.max(err / bnd)))
    # the first row: lambda_T is the jump at T
    jT = jump_of(S, [ckpt[S, c].astype(LD) for c in range(D)])
    for c in range(D):
        want = np.zeros(adj.shape[-1], dtype=LD) if jT is None else np.asarray(jT[c], dtype=LD)
        err = np.abs(np.asarray(adj[S - 1, 0, c].astype(LD) - want, dtype=np.float64))
        bnd = 4 * eps * np.abs(np.asarray(want, dtype=np.float64)) + 1e-300
        assert (err <= bnd).all(), (tag, c)


QUAD_RUNS = [  # family, shared p, dt, cost ("affine" / "explicit"), continuous cost (a, b) or None, no_start, saves
    ("lv", True, 0.1, "affine", None, False, "grid"), ("lv", False, 0.05, "explicit", None, True, "grid"),
    ("lv", True, 0.1, "affine", (0.5, -0.25), False, "sparse"), ("lorenz", False, 0.025, "affine", None, False, "grid"),
    ("robertson", True, 0.05, "explicit", (1.0, 0.0), True, "sparse")]


@pytest.mark.gpu
@pytest.mark.parametrize("family,shared_p,dt,cost,cont,no_start,saves", QUAD_RUNS)
def test_every_quadrature_reverse_row(probe, family, shared_p, dt, cost, cont, no_start, saves):
    import scimlsensitivity_jl_b200 as b
    N = 37
    T, u0, p = t5_problem(family, N, shared_p)
    S = int(round(T / dt))
    grid = np.arange(S + 1) * dt
    saveat = grid[::2] if saves == "grid" else np.array([grid[3], grid[S // 2], grid[S]])
    K = len(saveat)
    ca, cb = 1.0, -0.5
    eng = b.DeviceEnsemble(family, "quadrature", "tsit5_fixed", N, saveat, (0.0, T), dt, shared_p=shared_p,
                           cost=b.AffineCost(ca, cb) if cost == "affine" else None, no_start=no_start, quad_abstol=1e-10, quad_reltol=1e-10)
    if cont:
        eng.handle.set_continuous_cost(1, *cont)
    _, status = eng.forward(u0, p)
    assert (np.asarray(status) == 0).all()
    rng = np.random.default_rng(9)
    dLdu = rng.standard_normal((K, eng.d, N)) if cost == "explicit" else None
    du0, _ = eng.reverse(dLdu)
    S_, _, ckpt, adj = buffers_of(probe, eng, reverse=True)
    eng.close()
    assert S_ == S
    sos = {int(round(t / dt)): k for k, t in enumerate(saveat)}

    def jump_of(n, un):
        if n not in sos:
            return None
        if cost == "explicit":
            return [dLdu[sos[n], c] for c in range(len(un))]
        return [LD(ca) * un[c] + LD(cb) for c in range(len(un))]
    pm = member_params(p, shared_p, N, "f64")
    check_quad_rows(family, ckpt, adj, np.asarray(du0), S, dt, pm, jump_of, cont, no_start, f"{family} {cost} cont={cont} no_start={no_start}")
    print(f"quadrature rows {family} shared={shared_p} {cost} cont={cont} no_start={no_start}: observed error / bound {OBS}")
