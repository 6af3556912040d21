"""The random numbers and every forward step of the SDE kernels (csrc/sde_em.cuh), through tests/csrc/sde_probe.cu and
the public API, against tests/sde_restatement.py.

* Random words: b200adj::philox4x32_10 bit-identical to the toolkit's curand_Philox4x32_10 on the same words, to the
  integer restatement, and to the published Random123 known answers; the generator's counter (member lo, member hi,
  step, pair) and key (seed lo, seed hi) with seeds whose high word is nonzero and members >= 2^32.
* Normals and exported increments: normal_pair and every (step, component, member) of get_noise at traj_offset 0, 7,
  2^32 - 3 (straddling the member's word boundary) and 2^40 against the restatement in long double, whose uniforms are
  the device's exactly.  The bound, from the CUDA C Programming Guide's double-precision ulp table: log 1 ulp, halved
  by the sqrt, plus the sqrt's 0.5 ulp: rad within 1 eps relative; sincospi 2 ulp of |c| <= 1; the product rad c
  0.5 ulp: |z - Z| <= 3.5 eps rad.  dW = sqrt(h) z adds 0.5 ulp for sqrt(h) and 0.5 for the product, so
  |dW - DW| <= 4.5 eps sqrt(h) rad; the tests use 6 eps sqrt(h) rad.  wiener_increment<M> for M = 1, 2, 3 is the
  device's own sqrt(h) z products bit for bit, component 2q from z0 and 2q + 1 from z1 of pair q (M = 3: pair 1 gives
  only its z0).
* Every forward step, saveat = the full grid: u_{n+1} against one EM or EulerHeun step taken in long double from the
  device's own u_n and exported dW_n, for both families, all three noise modes (regenerated, stored_noise, caller-supplied
  dW) and shared and per-member p.  Each step starts from the device's state, so the bound is a few ulps of the terms:
      EM:  |u_{n+1} - U| <= 4 eps (|u| + h F(u) + |g(u) dW|)                                            =: B(u)
      EH:  <= 6 eps (|u| + h (F(u) + F(ub)) + (|g(u)| + |g(ub)|) |dW|) + (h |J_f(ub)| + |dW| |dg/du(ub)|) B(u) / 2
  where F sums the magnitudes of the monomials of f (the rounding of one evaluation) and ub is the predictor, whose own
  rounding B(u) the Jacobians pass on.  A single different increment moves u_{n+1} by |g dW| ~ 1e-2 sqrt(h), 1e11
  bounds: the forward pass used exactly the exported increments.

Observed on an H100 80GB HBM3 (700 W power limit), largest error as a share of its bound: normal_pair 0.28, get_noise
0.20, forward steps EM 0.23 and EulerHeun 0.14; the Philox words bit-identical throughout.  The module took 12 s of host
time there.
"""
import ctypes as C
import os
import subprocess
import sys

import numpy as np
import pytest

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(HERE)
for d in (ROOT, HERE):
    if d not in sys.path:
        sys.path.insert(0, d)

import sde_restatement as R
from scimlsensitivity_jl_b200 import _lib

CSRC = os.path.join(ROOT, "scimlsensitivity.jl_b200", "csrc")
PROBE = os.path.join(HERE, "csrc", "sde_probe.cu")
LD = np.longdouble
EPS = 2.220446049250313e-16
KAT = [((0x00000000, 0x00000000, 0x00000000, 0x00000000), (0x00000000, 0x00000000), (0x6627e8d5, 0xe169c58d, 0xbc57ac4c, 0x9b00dbd8)),
       ((0xffffffff, 0xffffffff, 0xffffffff, 0xffffffff), (0xffffffff, 0xffffffff), (0x408f276d, 0x41c83b0e, 0xa20bc7c6, 0x6d5451fd)),
       ((0x243f6a88, 0x85a308d3, 0x13198a2e, 0x03707344), (0xa4093822, 0x299f31d0), (0xd16cfe09, 0x94fdcceb, 0x5001e420, 0x24126ea1))]
SEEDS = (0, 100, 20260923, 0x9E3779B97F4A7C15, 0xFFFFFFFF00000001)
MEMBERS = (0, 1, 7, 2 ** 32 - 3, 2 ** 32 - 1, 2 ** 32, 2 ** 32 + 5, 2 ** 40 + 3, 2 ** 63 + 11)
OBS = {}


def _seen(kind, err, bound):
    OBS[kind] = max(OBS.get(kind, 0.0), float(np.max(np.asarray(err, dtype=np.float64) / np.asarray(bound, dtype=np.float64))))
    print(f"OBSERVED {kind}: {OBS[kind]:.3g} of the bound")


@pytest.fixture(scope="session")
def sde_probe_so(tmp_path_factory):
    """sde_probe.cu built with the library's nvcc flags, once per session, outside the source tree."""
    so = str(tmp_path_factory.mktemp("sde_probe") / "libsde_probe.so")
    cmd = [_lib.nvcc_path(), "-gencode", "arch=compute_90a,code=sm_90a", "-O3", "-std=c++17", "-I", CSRC,
           "-Xcompiler", "-fPIC", "-shared", PROBE, "-o", so]
    res = subprocess.run(cmd, capture_output=True, text=True)
    assert res.returncode == 0, res.stdout[-3000:] + res.stderr[-3000:]
    return so


def test_sde_probe_compiles_for_sm90a(sde_probe_so):
    """No GPU needed: a header change that breaks the probe fails here."""
    assert C.CDLL(sde_probe_so).probe_sde_random
    assert np.finfo(LD).eps <= 1.1e-19


@pytest.fixture(scope="module")
def probe(sde_probe_so):
    lib = C.CDLL(sde_probe_so)
    vp = C.c_void_p
    lib.probe_sde_random.argtypes = [C.c_int, vp, vp, vp, vp, C.c_int, vp, vp, vp, vp, vp, vp, vp]
    lib.probe_sde_random.restype = C.c_int

    def run(ctr, key, seed, member, step, pair, sqrth):
        ctr, key = np.ascontiguousarray(ctr, dtype=np.uint32), np.ascontiguousarray(key, dtype=np.uint32)
        n, nz = len(ctr), len(seed)
        ours, theirs = np.zeros((n, 4), np.uint32), np.zeros((n, 4), np.uint32)
        ins = [np.ascontiguousarray(seed, dtype=np.uint64), np.ascontiguousarray(member, dtype=np.uint64),
               np.ascontiguousarray(step, dtype=np.uint32), np.ascontiguousarray(pair, dtype=np.uint32),
               np.ascontiguousarray(sqrth, dtype=np.float64)]
        z, w = np.zeros((nz, 2)), np.zeros((nz, 6))
        rc = lib.probe_sde_random(n, ctr.ctypes.data, key.ctypes.data, ours.ctypes.data, theirs.ctypes.data, nz,
                                  *[a.ctypes.data for a in ins], z.ctypes.data, w.ctypes.data)
        assert rc == 0, f"probe failed: cudaError {rc}"
        return ours, theirs, z, w
    return run


def _generator_cases():
    seed, member, step, pair = [], [], [], []
    for s in SEEDS:
        for m in MEMBERS:
            for n in (0, 1, 99, 2 ** 31 + 7):
                for q in (0, 1, 2):
                    seed.append(s), member.append(m), step.append(n), pair.append(q)
    return (np.array(seed, dtype=np.uint64), np.array(member, dtype=np.uint64), np.array(step, dtype=np.uint32),
            np.array(pair, dtype=np.uint32))


@pytest.mark.gpu
def test_philox_words_match_curand_the_restatement_and_the_known_answers(probe):
    seed, member, step, pair = _generator_cases()
    ctr = np.stack([member & np.uint64(0xFFFFFFFF), member >> np.uint64(32), step, pair], 1)
    key = np.stack([seed & np.uint64(0xFFFFFFFF), seed >> np.uint64(32)], 1)
    ctr = np.concatenate([np.array([k[0] for k in KAT], dtype=np.uint64), ctr])
    key = np.concatenate([np.array([k[1] for k in KAT], dtype=np.uint64), key])
    ours, theirs, _, _ = probe(ctr, key, [], [], [], [], [])
    assert np.array_equal(ours, theirs)
    rest = np.stack(R.philox4x32_10(ctr.T, key.T), 1)
    assert np.array_equal(ours.astype(np.uint64), rest)
    assert [tuple(int(x) for x in row) for row in ours[:3]] == [k[2] for k in KAT]
    gen = [int(x) for x in R.words(0, 0, 0, 0)]      # the generator's own word layout at its origin is the first KAT
    assert gen == [int(x) for x in ours[0]]


@pytest.mark.gpu
def test_normal_pairs_and_wiener_increment_layout(probe):
    seed, member, step, pair = _generator_cases()
    sqrth = np.full(len(seed), np.sqrt(0.025))
    _, _, z, w = probe(np.zeros((0, 4)), np.zeros((0, 2)), seed, member, step, pair, sqrth)
    Z0, Z1, rad = [], [], []
    for i in range(len(seed)):
        a, b_, r = R.normal_pair(int(seed[i]), np.array([member[i]]), int(step[i]), int(pair[i]), "ld")
        Z0.append(a[0]), Z1.append(b_[0]), rad.append(r[0])
    Z = np.stack([np.array(Z0), np.array(Z1)], 1)
    bound = 3.5 * EPS * np.array(rad, dtype=np.float64)[:, None]
    err = np.abs(z.astype(LD) - Z).astype(np.float64)
    _seen("normal_pair", err, bound)
    assert (err <= bound).all()
    # wiener_increment<M>: sqrt(h) z of the device's own normal_pair for pair 0 (and pair 1 for the third component)
    p0 = pair == 0
    sq = sqrth[p0]
    assert np.array_equal(w[p0, 0], sq * z[p0, 0])
    assert np.array_equal(w[p0, 1:3], sq[:, None] * z[p0, :])
    assert np.array_equal(w[p0, 3:5], sq[:, None] * z[p0, :])
    key = {(int(seed[i]), int(member[i]), int(step[i]), int(pair[i])): i for i in range(len(seed))}
    i1 = np.array([key[(int(seed[i]), int(member[i]), int(step[i]), 1)] for i in np.nonzero(p0)[0]])
    assert np.array_equal(w[p0, 5], sq * z[i1, 0])


@pytest.mark.gpu
@pytest.mark.parametrize("traj_offset", [0, 7, 2 ** 32 - 3, 2 ** 40])
def test_exported_increments_against_the_restatement(traj_offset):
    import scimlsensitivity_jl_b200 as b
    N, S, h, seed = 8, R.S_STEPS, R.H, 0x9E3779B97F4A7C15
    eng = b.DeviceEnsemble("sde_lv", "backsolve", "em", N, R.GRID, (0.0, R.T_END), h, seed=seed, traj_offset=traj_offset)
    eng.forward(np.ones((2, N)), np.array(R.P_NOMINAL["sde_lv"]))
    dW = np.array(eng.noise())
    eng.close()
    DW, rad = R.increments(seed, traj_offset, N, S, 2, h, "ld")
    bound = 6 * EPS * np.sqrt(h) * rad.astype(np.float64)
    err = np.abs(dW.astype(LD) - DW).astype(np.float64)
    _seen("get_noise", err, bound)
    assert (err <= bound).all()


def _f_abs(family, u, p):
    if family == "sde_lv":
        return [abs(p[0] * u[0]) + abs(p[1] * u[0] * u[1]), abs(p[2] * u[1]) + abs(p[3] * u[0] * u[1])]
    return [abs(p[0] * u[0]), abs(p[0] * u[1])]


def _jac_abs_times(fn, y, p, v, diag=False):
    """|dfn/du (y)| v by complex steps in float64 (magnitudes only); diag: the diagonal alone"""
    yc = [np.asarray(x, dtype=np.complex128) for x in y]
    pc = [np.asarray(x, dtype=np.complex128) for x in p]
    out = [np.zeros(np.shape(y[0])) for _ in y]
    for c in range(len(y)):
        yy = list(yc)
        yy[c] = yy[c] + 1e-30j
        col = fn(yy, pc)
        for r in range(len(y)):
            if not diag or r == c:
                out[r] = out[r] + np.abs(np.imag(col[r]) / 1e-30) * np.abs(v[c])
    return out


@pytest.mark.gpu
@pytest.mark.parametrize("family", ["sde_lv", "sde_linear"])
@pytest.mark.parametrize("stepper", ["em", "euler_heun"])
@pytest.mark.parametrize("noise", ["regen", "stored", "dW"])
@pytest.mark.parametrize("shared_p", [True, False])
def test_every_forward_step(family, stepper, noise, shared_p):
    import scimlsensitivity_jl_b200 as b
    f, g, D, P = R.FAMILIES[family]
    N, h = 96, R.H
    c = dict(family=family, p="shared" if shared_p else "member")
    u0, p, _, _, _ = R.problem(dict(c, cost="scalar", saveat="full"), N, seed=5)
    eng = b.DeviceEnsemble(family, "backsolve", stepper, N, R.GRID, (0.0, R.T_END), h, shared_p=shared_p, seed=31,
                           traj_offset=2 ** 32 - 40, stored_noise=noise == "stored", cost=b.AffineCost(1.0, 0.0))
    dW_in = np.sqrt(h) * np.random.default_rng(2).standard_normal((R.S_STEPS, 2, N)) if noise == "dW" else None
    saved, status = eng.forward(u0, p, dW=dW_in)
    saved, dW = np.array(saved), np.array(eng.noise())
    eng.close()
    assert (np.asarray(status) == 0).all()
    if dW_in is not None:
        assert np.array_equal(dW, dW_in)
    pm = np.asarray(p, dtype=np.float64)
    pm = np.repeat(pm[:, None], N, 1) if pm.ndim == 1 else pm
    pl = [x.astype(LD) for x in pm]
    assert np.array_equal(saved[0], u0)
    worst = 0.0
    for n in range(R.S_STEPS):
        u, w = [x.astype(LD) for x in saved[n]], [x.astype(LD) for x in dW[n]]
        U = R.forward(R.Kind("ld"), family, stepper, u, pl, [w], LD(h))[1]
        err = np.abs(saved[n + 1].astype(LD) - np.array(U)).astype(np.float64)
        u64, w64 = saved[n], dW[n]
        F, gv = _f_abs(family, u64, pm), g(u64, pm)
        B = [4 * EPS * (np.abs(u64[j]) + h * F[j] + np.abs(gv[j] * w64[j])) for j in range(D)]
        if stepper == "em":
            bound = np.array(B)
        else:
            fv = f(u64, pm)
            ub = [u64[j] + h * fv[j] + gv[j] * w64[j] for j in range(D)]
            Fb, gb = _f_abs(family, ub, pm), g(ub, pm)
            Jf = _jac_abs_times(f, ub, pm, B)
            Jg = _jac_abs_times(g, ub, pm, [np.abs(w64[j]) * B[j] for j in range(D)], diag=True)
            bound = np.array([6 * EPS * (np.abs(u64[j]) + h * (F[j] + Fb[j]) + (np.abs(gv[j]) + np.abs(gb[j])) * np.abs(w64[j]))
                              + 0.5 * (h * Jf[j] + Jg[j]) for j in range(D)])
        worst = max(worst, float((err / bound).max()))
        assert (err <= bound).all(), (n, float((err / bound).max()))
    _seen(f"forward {stepper}", worst, 1.0)
