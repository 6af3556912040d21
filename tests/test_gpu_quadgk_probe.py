"""The warp-cooperative quadgk of QuadratureAdjoint (csrc/quadgk.cuh), one part at a time, through tests/csrc/quadgk_probe.cu:
the production device functions wrapped in one-warp kernels (and one persistent-grid kernel for the member loop).

* `coop_count` (the interval lookup inside a segment's index brackets) exactly against numpy.searchsorted, for the scanned
  (<= 6 knots), lane-bisected (<= 32) and strided (> 32) windows, ascending and descending.
* `warp_argmax_lane` and the queue arg-max exactly: ties resolve to the lowest segment index, as the oracle's linear scan.
* `quadgk_warp` against an fp64 restatement of the QuadGK adapt loop (itself pinned against the oracle's `oracle_quadgk`) and
  against exact integrals: same segment count, bitwise equal segment ends (they are dyadic), the integral within 1e-13 of
  the restatement.  Step integrands drive the queue through the block-maxima path (> 32 segments), global keys (> 512),
  several blocks per lane (> 1024) and the capacity limit.
* the block-maxima table of a warp holds ceil(maxseg / 32) entries (a partial last block included); the probes' shared
  allocations end in a sentinel guard region, so a store past the table is observed, never a fault.
* `quad_member_loop` (scratch reused from member to member): every member's result bitwise equal to that member alone.
* the production integrand contexts (RosQuadCtx, T5aQuadCtx) on synthetic records: every lookup checked against a scan of
  all knots, the integral against the exact piecewise integral.

Cost: the fp64 restatement takes at most 0.5 s of host time per run (4336 segments, P = 4), the exact piecewise integral of
the 8000-knot layout 2 s; the whole module ran in 35 s on an H100 SXM (700 W), the probe's compilation 8 s of it.
Two changes to coop_count cannot be observed and so are not pinned: where the scan of a <= 32-knot window hands over to the
lane bisection (both count exactly for any window), and hi = lo + stride - 1 in the wide search (the answer never exceeds
it: below the last full stride, the uncounted sample at lo + stride - 1 bounds the answer; past it, the tail holds fewer
than `stride` knots, so cnt <= lo + stride - 1).
"""
import ctypes as C
import math
import os
import subprocess
from fractions import Fraction

import numpy as np
import pytest

from scimlsensitivity_jl_b200 import _lib

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
CSRC = os.path.join(ROOT, "scimlsensitivity.jl_b200", "csrc")
PROBE = os.path.join(ROOT, "tests", "csrc", "quadgk_probe.cu")

# Gauss-Kronrod (7, 15): abscissae of the 15-point Kronrod rule (x_0 .. x_7 = 0), its weights, the 7-point Gauss weights
XGK = [0.991455371120812639206854697526329, 0.949107912342758524526189684047851, 0.864864423359769072789712788640926,
       0.741531185599394439863864773280788, 0.586087235467691130294144838258730, 0.405845151377397166906606412076961,
       0.207784955007898467600689403773245, 0.0]
WGK = [0.022935322010529224963732008058970, 0.063092092629978553290700663189204, 0.104790010322250183839876322541518,
       0.140653259715525918745189590510238, 0.169004726639267902826583426598550, 0.190350578064785409913256402421014,
       0.204432940075298892414161999234649, 0.209482141084727828012999174891714]
WG = [0.129484966168869693270611432679082, 0.279705391489276667901467771423780, 0.381830050505118944950369775488975,
      0.417959183673469387755102040816327]
GUARD_PAD = 64          # quadgk_probe.cu: PAD extra segment records after maxseg


# ------------------------------------------------------------------------------------------------------------------------
# the reference: QuadGK's adapt loop restated in fp64 (the oracle's order of operations), and exact integrals


def _gk15(f, a, b, P, jt=None):
    """-> (I[P], err, min distance of a node to a jump in ulps) of the (7, 15) pair on [a, b]"""
    c, hl = 0.5 * (a + b), 0.5 * (b - a)
    x = np.array(XGK[:7])
    tl, tr = c - hl * x, c + hl * x
    v = f(np.concatenate([[c], tl, tr]))
    fc, fl, fr = v[0], v[1:8], v[8:15]
    Ik = WGK[7] * fc
    Ig = WG[3] * fc
    for j in range(7):
        s = fl[j] + fr[j]
        Ik = Ik + WGK[j] * s
        if j & 1:
            Ig = Ig + WG[j // 2] * s
    Ik, Ig = Ik * hl, Ig * hl
    e2 = 0.0
    for q in range(P):
        d = float(Ik[q] - Ig[q])
        e2 += d * d
    near = math.inf
    if jt is not None and len(jt):          # the centre node c is computed exactly on both sides; the others may round apart
        nodes = np.concatenate([tl, tr])
        near = float(np.min(np.abs(nodes[:, None] - jt[None, :]) / np.spacing(np.abs(nodes))[:, None]))
    return Ik, math.sqrt(e2), near


def quadgk_ref(f, P, a, b, atol, rtol, maxseg, jt=None):
    """QuadGK's adapt loop: pop the largest error (ties -> lowest index), bisect at 0.5 (a + b), update the running totals
    incrementally, give up (ok = False) when a bisection would need segment maxseg + 1.  f(t[n]) -> [n][P].
    -> dict(I, ok, nseg, segs[nseg][2], margin = closest |E - tol| / tol of any stopping test, near = closest node-to-jump
    distance in ulps)."""
    segs = np.zeros((max(maxseg, 1) + 1, 2))
    errs = np.full(max(maxseg, 1) + 1, -1.0)
    Is = np.zeros((max(maxseg, 1) + 1, P))
    I0, e0, near = _gk15(f, a, b, P, jt)
    segs[0], errs[0], Is[0] = (a, b), e0, I0
    Itot, E, n, ok, margin = I0.copy(), e0, 1, True, math.inf
    while True:
        nI = 0.0
        for q in range(P):
            nI += float(Itot[q]) * float(Itot[q])
        tol = max(atol, rtol * math.sqrt(nI))
        margin = min(margin, abs(E - tol) / tol if tol > 0 else (math.inf if E == 0 else 0.0))
        if E <= tol:
            break
        if n + 1 > maxseg:
            ok = False
            break
        w = int(np.argmax(errs[:n]))
        aw, bw = segs[w]
        mid = 0.5 * (aw + bw)
        if not (min(aw, bw) < mid < max(aw, bw)):
            break
        Il, el, n1 = _gk15(f, aw, mid, P, jt)
        Ir, er, n2 = _gk15(f, mid, bw, P, jt)
        near = min(near, n1, n2)
        E += (el + er) - errs[w]
        Itot = Itot + ((Il + Ir) - Is[w])
        segs[w], errs[w], Is[w] = (aw, mid), el, Il
        segs[n], errs[n], Is[n] = (mid, bw), er, Ir
        n += 1
    return {"I": Itot, "ok": ok, "nseg": n, "segs": segs[:n].copy(), "margin": margin, "near": near}


def step_fn(jt, js, scale=1.0):
    """f_q(t) = scale * sum_j js[j][q] [t >= jt[j]], jt ascending: the device's sequential sum over j is a prefix sum"""
    cs = np.cumsum(js, axis=0)

    def f(t):
        k = np.searchsorted(jt, t, side="right")
        out = np.where(k[:, None] > 0, cs[np.maximum(k - 1, 0)], 0.0)
        return out * scale
    return f


def step_exact(jt, js, a, b, scale=1):
    """exact integral of the step function over [a, b] (rational arithmetic)"""
    A, B = Fraction(a), Fraction(b)
    return [float(Fraction(scale) * sum(Fraction(float(js[j, q])) * (B - min(max(Fraction(float(jt[j])), A), B)) for j in range(len(jt))))
            for q in range(js.shape[1])]


def poly_fn(c):
    def f(t):
        return np.stack([np.polynomial.polynomial.polyval(t, c[q]) for q in range(c.shape[0])], axis=1)
    return f


def poly_exact(c, a, b):
    A, B = Fraction(a), Fraction(b)
    return [float(sum(Fraction(float(c[q, k])) * (B ** (k + 1) - A ** (k + 1)) / (k + 1) for k in range(c.shape[1]))) for q in range(c.shape[0])]


def make_steps(seed, nj, P, a=-1.0, b=3.0, ndyadic=None):
    """nj jumps of distinct sizes in (a, b): about a third exactly on bisection points of [a, b], the rest at random
    (non-dyadic) points.  -> jt ascending, js[nj][P]"""
    rng = np.random.default_rng(seed)
    nd = nj // 3 if ndyadic is None else ndyadic
    m = rng.integers(1, 9, nd)
    dy = a + (b - a) * (2 * rng.integers(0, 2 ** (m - 1)) + 1) / 2.0 ** m
    jt = np.concatenate([np.unique(dy), rng.uniform(a, b, nj - len(np.unique(dy)))])
    order = np.argsort(jt)
    js = rng.uniform(0.5, 2.0, (nj, P)) * rng.choice([-1.0, 1.0], (nj, P))
    return jt[order], js


# step integrands on [-1, 3] (seed, jumps, atol) tuned to the segment counts named; P = 1 unless stated
STEP_CASES = {"s20": (1, 2, 1e-4), "s40": (2, 3, 1e-7), "s600": (3, 40, 1e-6), "s1500": (4, 120, 1e-6), "s4000": (5, 260, 1e-7)}


# ------------------------------------------------------------------------------------------------------------------------
# CPU: the restatement against the oracle


def _oracle_quadgk(f, P, a, b, atol, rtol):
    from oracle import oracle as O
    lib = O.lib()
    FN = C.CFUNCTYPE(None, C.c_double, C.POINTER(C.c_double), C.c_void_p)

    def cb(t, out, ctx):
        v = f(np.array([t]))[0]
        for q in range(P):
            out[q] = float(v[q])
    fn = FN(cb)
    lib.oracle_quadgk.argtypes = [FN, C.c_void_p, C.c_int, C.c_double, C.c_double, C.c_double, C.c_double, C.POINTER(C.c_double)]
    lib.oracle_quadgk.restype = C.c_long
    out = (C.c_double * P)()
    evals = lib.oracle_quadgk(fn, None, P, a, b, atol, rtol, out)
    assert (evals - 15) % 30 == 0
    return np.array(out[:]), 1 + (evals - 15) // 30


@pytest.mark.parametrize("case", ["s40", "s600", "poly_p3", "s20_p4"])
def test_restatement_matches_the_oracle(case):
    if case == "poly_p3":
        c = np.random.default_rng(7).standard_normal((3, 24))
        f, P, a, b, atol, rtol = poly_fn(c), 3, -0.3, 1.7, 0.0, 1e-14
    else:
        name, P = (case[:-3], 4) if case.endswith("_p4") else (case, 1)
        seed, nj, atol = STEP_CASES[name]
        jt, js = make_steps(seed, nj, P)
        f, a, b, rtol = step_fn(jt, js), -1.0, 3.0, 0.0
    ref = quadgk_ref(f, P, a, b, atol, rtol, 1 << 20)
    I, n = _oracle_quadgk(f, P, a, b, atol, rtol)
    assert n == ref["nseg"]
    assert np.abs(I - ref["I"]).max() <= 1e-15 * np.abs(ref["I"]).max()


# ------------------------------------------------------------------------------------------------------------------------
# the probe library


@pytest.fixture(scope="session")
def probe_so(tmp_path_factory):
    """quadgk_probe.cu built with the library's own nvcc flags, once per session, outside the source tree."""
    so = str(tmp_path_factory.mktemp("quadgk_probe") / "libquadgk_probe.so")
    cmd = [_lib.nvcc_path(), "-gencode", "arch=compute_90a,code=sm_90a", "-O3", "-std=c++17", "-I", CSRC,
           "-Xcompiler", "-fPIC", "-shared", PROBE, "-o", so]
    res = subprocess.run(cmd, capture_output=True, text=True)
    assert res.returncode == 0, res.stdout[-3000:] + res.stderr[-3000:]
    return so


def test_probe_compiles_for_sm90a(probe_so):
    """No GPU needed: a header change that breaks the probes fails here."""
    lib = C.CDLL(probe_so)
    for name in ("probe_layout", "probe_coop_count", "probe_warp_argmax", "probe_queue_argmax", "probe_quadgk", "probe_member_loop", "probe_ctx"):
        getattr(lib, name)


@pytest.mark.parametrize("maxseg", [100, 400, 2000, 4096, 16382, 16384])
def test_block_maxima_table_covers_every_key(probe_so, maxseg):
    """Key maxseg - 1 lies in block (maxseg - 1) // 32: a warp needs ceil(maxseg / 32) block maxima, and the dynamic shared
    memory of a quadrature block holds QUAD_WARPS of those tables after the QUAD_WARPS x QUAD_SKEYS shared keys."""
    lib = C.CDLL(probe_so)
    sm, l1, warps, skeys = C.c_longlong(), C.c_int(), C.c_int(), C.c_int()
    lib.probe_layout(maxseg, C.byref(sm), C.byref(l1), C.byref(warps), C.byref(skeys))
    need = -(-maxseg // 32)
    assert l1.value == need
    assert (maxseg - 1) // 32 < l1.value
    assert sm.value == warps.value * (skeys.value + need) * 8


@pytest.fixture(scope="module")
def probe(probe_so):
    lib = C.CDLL(probe_so)
    vp, i, d = C.c_void_p, C.c_int, C.c_double
    lib.probe_coop_count.argtypes = [i, vp, i, i, vp, vp]
    lib.probe_warp_argmax.argtypes = [vp, vp, vp]
    lib.probe_queue_argmax.argtypes = [vp, vp, vp, i, vp, vp, vp]
    lib.probe_quadgk.argtypes = [i, i, d, d, d, d, i, i, vp, i, vp, vp, d, vp, vp, vp, vp]
    lib.probe_member_loop.argtypes = [i, C.c_longlong, i, vp, d, d, d, d, i, vp, vp, vp, vp, vp, vp, vp, vp, vp]
    lib.probe_ctx.argtypes = [i, vp, vp, vp, vp, vp, vp, i, i, d, d, d, d, i, vp, vp, vp]
    return lib


def _dev(x, dtype=None):
    import torch
    x = np.ascontiguousarray(x)
    if dtype is None:
        dtype = torch.float64 if x.dtype.kind == "f" else torch.int32
    return torch.tensor(x, dtype=dtype, device="cuda")


def _check(rc):
    assert rc == 0, f"probe launch failed: cudaError {rc}"


# ------------------------------------------------------------------------------------------------------------------------
# coop_count


def _coop(probe, knots, first, cnt, t, asc):
    import torch
    kd, td = _dev(knots), _dev(t)
    out = torch.full((32,), -7, dtype=torch.int32, device="cuda")
    _check(probe.probe_coop_count(int(asc), kd.data_ptr(), first, cnt, td.data_ptr(), out.data_ptr()))
    return out.cpu().numpy()


def _probe_points(sub, rng):
    """values of t: below / above the window, on every knot, one ulp either side of a knot, random interior points"""
    lo, hi = sub.min(), sub.max()
    pts = [lo - 1.0, np.nextafter(lo, -np.inf), hi + 1.0, np.nextafter(hi, np.inf)]
    pts += list(sub)
    pts += list(np.nextafter(sub, np.inf)) + list(np.nextafter(sub, -np.inf))
    pts += list(rng.uniform(lo, hi, 32))
    pts = np.array(pts, dtype=np.float64)
    return pts


@pytest.mark.gpu
@pytest.mark.parametrize("asc", [True, False], ids=["asc", "desc"])
@pytest.mark.parametrize("cnt", [0, 1, 2, 5, 6, 7, 8, 31, 32, 33, 63, 64, 65, 1023, 1024, 1025, 4097])
def test_coop_count_is_searchsorted(probe, cnt, asc):
    rng = np.random.default_rng(1000 + cnt + (0 if asc else 1))
    first = 3 + cnt % 5
    n = first + cnt + 7
    # Robertson-like geometric knots over 1e-8 .. 1e2 with duplicated knots (zero-length steps)
    base = np.geomspace(1e-8, 1e2, max(n, 2))[:n]
    if n > 4:
        dup = rng.choice(np.arange(1, n - 1), size=max(1, n // 9), replace=False)
        base[dup] = base[dup - 1]
    knots = np.sort(base) if asc else np.sort(base)[::-1].copy()
    sub = knots[first:first + cnt]
    pts = _probe_points(sub, rng) if cnt else np.array([0.5, -1.0, 1e3])
    pts = np.concatenate([pts, np.zeros((-len(pts)) % 32)])
    for k in range(0, len(pts), 32):
        t = pts[k:k + 32]
        got = _coop(probe, knots, first, cnt, t, asc)
        want = np.searchsorted(sub, t, side="left") if asc else np.searchsorted(-sub, -t, side="left")
        assert np.array_equal(got, want), f"cnt {cnt} asc {asc}: t {t[got != want][:4]} got {got[got != want][:4]} want {want[got != want][:4]}"


# ------------------------------------------------------------------------------------------------------------------------
# arg-max


def _bits_argmax(v, present):
    """lowest lane among the present lanes holding the largest value (non-negative doubles: the order of their bits)"""
    bits = np.where(present, v.view(np.int64), -1)
    return int(np.argmax(bits)) if present.any() else -1


@pytest.mark.gpu
def test_warp_argmax_lane(probe):
    import torch
    rng = np.random.default_rng(5)
    sub = np.array([5e-324, 1e-310, 2.2250738585072014e-308])
    cases = []
    v = rng.uniform(0, 1, 32); v[7] = v[21] = 2.0; cases.append((v, np.ones(32, bool)))                      # tie
    v = np.full(32, 1.5); v[9] = np.nextafter(1.5, 2.0); v[30] = np.nextafter(v[9], 2.0); cases.append((v, np.ones(32, bool)))  # low word
    v = np.zeros(32); cases.append((v, np.ones(32, bool)))                                                    # all 0.0
    v = np.zeros(32); v[[3, 17, 29]] = sub; cases.append((v, np.ones(32, bool)))                             # subnormals
    v = np.zeros(32); v[4] = sub[0]; cases.append((v, np.ones(32, bool)))
    v = rng.uniform(0, 1, 32); v[0] = 9.0; pr = np.ones(32, bool); pr[0] = False; cases.append((v, pr))      # masked winner
    v = rng.uniform(0, 1, 32); pr = np.zeros(32, bool); pr[[12, 13]] = True; v[12] = v[13]; cases.append((v, pr))
    v = np.zeros(32); pr = np.zeros(32, bool); pr[31] = True; cases.append((v, pr))
    v = rng.uniform(0, 1, 32); cases.append((v, np.zeros(32, bool)))                                         # nobody present
    for v, pr in cases:
        vd, pd = _dev(v), _dev(pr.astype(np.int32))
        out = torch.full((32,), -9, dtype=torch.int32, device="cuda")
        _check(probe.probe_warp_argmax(vd.data_ptr(), pd.data_ptr(), out.data_ptr()))
        got = out.cpu().numpy()
        assert (got == got[0]).all()
        assert got[0] == _bits_argmax(v, pr), (v, pr, got[0])


def _queue_argmax(probe, keys):
    """run the production queue arg-max over keys[0 .. n-1]: shared keys below QUAD_SKEYS, global keys from there; every slot
    the production code must not read holds a poison larger than any key"""
    import torch
    n = len(keys)
    poison = 1e300
    skey = np.full(512, poison); skey[:min(n, 512)] = keys[:512]
    key = np.full(n + GUARD_PAD, poison); key[512:n] = keys[512:]
    nb = -(-n // 32)
    l1 = np.array([keys[32 * b:32 * b + 32].max() for b in range(nb)])
    ts = [_dev(skey), _dev(key), _dev(l1)]
    w = torch.full((2,), -1, dtype=torch.int32, device="cuda")
    ew = torch.zeros(1, dtype=torch.float64, device="cuda")
    g = torch.zeros(1, dtype=torch.int32, device="cuda")
    _check(probe.probe_queue_argmax(ts[0].data_ptr(), ts[1].data_ptr(), ts[2].data_ptr(), n, w.data_ptr(), ew.data_ptr(), g.data_ptr()))
    assert g.item() == 1
    return int(w[0].item()), int(w[1].item()), float(ew.item())


def _queue_cases():
    rng = np.random.default_rng(11)
    cases = {}
    k = rng.uniform(0, 1, 100); k[[40, 45]] = 3.0; cases["tie_in_block"] = k
    k = np.full(70, 1.0); k[[5, 66]] = np.nextafter(1.0, 2.0); cases["low_word"] = k
    k = np.zeros(64); cases["all_zero"] = k
    k = np.zeros(96); k[[33, 70]] = 5e-324; cases["subnormal_tie"] = k
    # > 32 blocks: equal maxima in blocks b and b + 32 (lane b scans both); the lower block must win
    for b in (0, 1, 7, 31):
        k = rng.uniform(0, 1, 2100); k[32 * b + 5] = k[32 * (b + 32) + 3] = 4.0
        if b == 1:
            k[32 * 32 + 9] = 4.0          # block 32, held by lane 0, ties too
        cases[f"blocks_{b}_and_{b + 32}"] = k
    k = rng.uniform(0, 1, 4000); k[[3000, 130, 3999]] = 6.0; cases["three_way_tie_global"] = k
    # either side of QUAD_SKEYS = 512
    for w in (511, 512, 513):
        k = rng.uniform(0, 1, 600); k[w] = 2.0; cases[f"max_at_{w}"] = k
    k = rng.uniform(0, 1, 600); k[511] = k[512] = 2.0; cases["tie_511_512"] = k
    k = rng.uniform(0, 1, 513); k[512] = 2.0; cases["nseg_513"] = k
    return cases


@pytest.mark.gpu
@pytest.mark.parametrize("case", list(_queue_cases()))
def test_queue_argmax_is_the_lowest_index_maximum(probe, case):
    keys = _queue_cases()[case]
    w, bi, ew = _queue_argmax(probe, keys)
    want = int(np.argmax(keys))           # first maximum, as the oracle's linear scan
    assert (w, bi) == (want, want // 32), f"{case}: segment {w} (block {bi}), expected {want}"
    assert ew == keys[want]


# ------------------------------------------------------------------------------------------------------------------------
# quadgk_warp


def _run_quadgk(probe, P, a, b, atol, rtol, maxseg, kind=1, jt=None, js=None, coef=None, tnan=0.0):
    import torch
    zero = _dev(np.zeros(1))
    jtd = _dev(jt) if jt is not None else zero
    jsd = _dev(js.ravel()) if js is not None else zero
    cd = _dev(coef.ravel()) if coef is not None else zero
    deg = coef.shape[1] - 1 if coef is not None else 0
    calls = torch.zeros(1, dtype=torch.int32, device="cuda")
    out = torch.full((P,), float("nan"), dtype=torch.float64, device="cuda")
    info = torch.full((3,), -1, dtype=torch.int32, device="cuda")
    ab = torch.full(((maxseg + GUARD_PAD) * 2,), float("nan"), dtype=torch.float64, device="cuda")
    _check(probe.probe_quadgk(kind, P, a, b, atol, rtol, maxseg, deg, cd.data_ptr(), 0 if jt is None else len(jt), jtd.data_ptr(),
                              jsd.data_ptr(), tnan, calls.data_ptr(), out.data_ptr(), info.data_ptr(), ab.data_ptr()))
    ok, n, guard = (int(x) for x in info.cpu().numpy())
    return {"I": out.cpu().numpy(), "ok": bool(ok), "nseg": n, "guard": bool(guard), "segs": ab.cpu().numpy()[:2 * n].reshape(n, 2)}


@pytest.mark.gpu
@pytest.mark.parametrize("P", [1, 3, 4, 8])
@pytest.mark.parametrize("deg", [13, 22])
def test_quadgk_polynomials_in_one_segment(probe, P, deg):
    """G7 is exact to degree 13 and K15 to degree 22: one segment, and the integral to about 1e-15.  Pins the nodes, the
    weights, the lane-to-node map and the shuffle reduction of gk15_pair for every P."""
    c = np.random.default_rng(100 * P + deg).standard_normal((P, deg + 1))
    a, b = -0.3, 1.7
    exact = np.array(poly_exact(c, a, b))
    # degree 22: G7 is not exact, so the tolerance accepts the first segment's estimate (twice the restatement's)
    atol = 2 * _gk15(poly_fn(c), a, b, P)[1] if deg == 22 else 1e-12
    assert quadgk_ref(poly_fn(c), P, a, b, atol, 0.0, 64)["nseg"] == 1
    r = _run_quadgk(probe, P, a, b, atol, 0.0, 64, kind=0, coef=c)
    assert r["ok"] and r["nseg"] == 1 and r["guard"]
    scale = np.abs(exact).max()
    err = np.abs(r["I"] - exact).max() / scale
    assert err <= 4e-15, f"P {P} degree {deg}: relative error {err:.2e}"
    print(f"degree {deg} P {P}: relative error {err:.1e}")


def _step_case(name, P):
    seed, nj, atol = STEP_CASES[name]
    jt, js = make_steps(seed, nj, P)
    return jt, js, atol


def _compare(r, ref, exact, atol, rtol):
    """Same segment count, bitwise equal ends, the integral within 1e-13 of the restatement.  Against the exact integral:
    within max(atol, rtol |I|) where the restatement is; QuadGK's error estimate is not a bound for a step function (a jump
    between a segment's outermost node and its end is invisible to both rules: estimate 0, error up to 0.0086 hl |jump|),
    and there the device must carry exactly the restatement's error."""
    assert r["nseg"] == ref["nseg"], f"segments {r['nseg']} vs restatement {ref['nseg']}"
    assert r["ok"] == ref["ok"]
    assert np.array_equal(r["segs"], ref["segs"]), "final segment ends differ"
    scale = np.abs(ref["I"]).max()
    assert np.abs(r["I"] - ref["I"]).max() <= 1e-13 * scale
    tol = max(atol, rtol * np.linalg.norm(exact))
    err_ref = np.abs(ref["I"] - exact).max()
    assert np.abs(r["I"] - exact).max() <= (tol if err_ref <= tol else err_ref + 1e-13 * scale)


@pytest.mark.gpu
@pytest.mark.parametrize("P", [1, 3, 4, 8])
@pytest.mark.parametrize("name", list(STEP_CASES))
def test_quadgk_step_functions_match_the_restatement(probe, name, P):
    if P == 8 and name == "s4000":
        pytest.skip("covered by P = 1, 3, 4")
    jt, js, atol = _step_case(name, P)
    a, b, maxseg = -1.0, 3.0, 8192
    ref = quadgk_ref(step_fn(jt, js), P, a, b, atol, 0.0, maxseg, jt)
    assert ref["near"] > 8 and ref["margin"] > 1e-9, "test construction: a node or the stopping test is within rounding of a decision"
    r = _run_quadgk(probe, P, a, b, atol, 0.0, maxseg, jt=jt, js=js)
    assert r["guard"]
    exact = np.array(step_exact(jt, js, a, b))
    _compare(r, ref, exact, atol, 0.0)
    print(f"{name} P {P}: {r['nseg']} segments, |I - restatement| {np.abs(r['I'] - ref['I']).max():.1e}, |I - exact| {np.abs(r['I'] - exact).max():.1e}")


# ------------------------------------------------------------------------------------------------------------------------
# capacity and the block-maxima table


@pytest.mark.gpu
@pytest.mark.parametrize("name", ["s20", "s600"])
def test_quadgk_capacity_limit(probe, name):
    """maxseg = what the integrand needs: the same run; one less: ok = False (and NaN through the member loop)."""
    jt, js, atol = _step_case(name, 1)
    f = step_fn(jt, js)
    need = quadgk_ref(f, 1, -1.0, 3.0, atol, 0.0, 1 << 20, jt)["nseg"]
    r = _run_quadgk(probe, 1, -1.0, 3.0, atol, 0.0, need, jt=jt, js=js)
    assert r["ok"] and r["nseg"] == need and r["guard"] and np.isfinite(r["I"]).all()
    r = _run_quadgk(probe, 1, -1.0, 3.0, atol, 0.0, need - 1, jt=jt, js=js)
    assert not r["ok"] and r["nseg"] == need - 1 and r["guard"]
    js3 = np.repeat(js, 3, axis=1)                  # the member loop integrates P = 3 components
    need3 = quadgk_ref(step_fn(jt, js3), 3, -1.0, 3.0, atol, 0.0, 1 << 20, jt)["nseg"]
    for maxseg, finite in ((need3, True), (need3 - 1, False)):
        dp = _member_loop(probe, [(jt, js3)], [0], np.array([1.0]), np.zeros(0), -1.0, 3.0, atol, 0.0, maxseg, grid=1)[0]
        assert np.isfinite(dp).all() == finite and (finite or np.isnan(dp).all())


@pytest.mark.gpu
def test_quadgk_nan_integrand_gives_nan(probe):
    """A NaN at one node of the root segment reaches the result: never a finite number."""
    c = np.random.default_rng(3).standard_normal((3, 6))
    a, b = -0.3, 1.7
    tnan = 0.5 * (a + b) + 0.5 * (b - a) * XGK[3]
    r = _run_quadgk(probe, 3, a, b, 1e-10, 0.0, 200, kind=2, coef=c, tnan=tnan)
    assert r["guard"] and np.isnan(r["I"]).all()


# integrands needing more than 32 floor(maxseg / 32) but at most maxseg segments: (seed, jumps, atol)
OVERFLOW_CASES = {400: (21, 30, 2.4887034759027854e-07), 2000: (22, 100, 1.3412717530678956e-09)}


@pytest.mark.gpu
@pytest.mark.parametrize("maxseg", list(OVERFLOW_CASES))
def test_partial_last_block_stays_inside_the_table(probe, maxseg):
    """Segments in the partial last block of keys (index >= 32 floor(maxseg / 32)) update a block maximum of their own;
    the shared table holds it and the guard after the table stays intact."""
    seed, nj, atol = OVERFLOW_CASES[maxseg]
    jt, js = make_steps(seed, nj, 1)
    ref = quadgk_ref(step_fn(jt, js), 1, -1.0, 3.0, atol, 0.0, maxseg, jt)
    assert 32 * (maxseg // 32) < ref["nseg"] <= maxseg and ref["ok"], f"test construction: {ref['nseg']} segments"
    r = _run_quadgk(probe, 1, -1.0, 3.0, atol, 0.0, maxseg, jt=jt, js=js)
    assert r["guard"], "store past the block-maxima table"
    _compare(r, ref, np.array(step_exact(jt, js, -1.0, 3.0)), atol, 0.0)


# ------------------------------------------------------------------------------------------------------------------------
# the member loop


def _member_loop(probe, sets, which, mult, saveat, t0, t1, atol, rtol, maxseg, grid):
    """member i integrates step set sets[which[i]] times mult[i] -> dp[P][N], calls[N], guard per block, and (K = 0) the
    number of block maxima that differ from the maxima of the keys each warp's last member left, at the quad_smem layout"""
    import torch
    N = len(which)
    jt = np.concatenate([s[0] for s in sets]); js = np.concatenate([s[1] for s in sets])
    offs = np.cumsum([0] + [len(s[0]) for s in sets])
    joff = np.array([offs[w] for w in which], np.int32); nj = np.array([len(sets[w][0]) for w in which], np.int32)
    keep = [_dev(joff), _dev(nj), _dev(np.asarray(mult, np.float64)), _dev(jt), _dev(js.ravel()), _dev(saveat if len(saveat) else np.zeros(1))]
    calls = torch.zeros(N, dtype=torch.int32, device="cuda")
    dp = torch.full((3, N), float("nan"), dtype=torch.float64, device="cuda")
    g = torch.zeros(grid, dtype=torch.int32, device="cuda")
    l1_bad = torch.zeros(1, dtype=torch.int32, device="cuda")
    _check(probe.probe_member_loop(grid, N, len(saveat), keep[5].data_ptr(), t0, t1, atol, rtol, maxseg, keep[0].data_ptr(), keep[1].data_ptr(),
                                   keep[2].data_ptr(), keep[3].data_ptr(), keep[4].data_ptr(), calls.data_ptr(), dp.data_ptr(), g.data_ptr(),
                                   l1_bad.data_ptr()))
    return dp.cpu().numpy(), calls.cpu().numpy(), g.cpu().numpy(), int(l1_bad.item())


def _intervals(saveat, t0, t1):
    """the data intervals in the order quad_member_loop integrates them"""
    K = len(saveat)
    if K == 0:
        return [(t0, t1)]
    iv = []
    if saveat[-1] != t1:
        iv.append((saveat[-1], t1))
    for k in range(K - 2, -1, -1):
        if saveat[k] != saveat[k + 1]:
            iv.append((saveat[k], saveat[k + 1]))
    if saveat[0] != t0:
        iv.append((t0, saveat[0]))
    return iv


# the two members of the loop test, both driven by rtol (atol = 0), so that a member's scale factor leaves its bisections
# unchanged: ~3000 segments (more than 32 floor(3100 / 32) = 3072 for K = 0) and a single jump on a bisection point
ML_BIG, ML_RTOL, ML_MAXSEG = (31, 130), 1.0803315190764665e-12, 3100
ML_SMALL = (np.array([2.0]), np.array([[0.7, -1.3, 0.4]]))
SAVEAT_CASES = {"K0": [], "duplicates": [0.375, 0.375, 1.25, 2.5, 2.5], "first_is_t0": [-1.0, 0.5, 2.0], "last_is_t1": [0.0, 1.5, 3.0],
                "both_ends": [-1.0, 1.0, 1.0, 3.0]}


def _member_kinds(N, G):
    """member i -> 0 (big) / 1 (small).  Warp g of G takes members g, g + G, ...; kinds alternate per ROUND, so every warp
    runs big, small, big, ...: a small member reuses the scratch a big one left, and the four warps of a block (the last
    one, whose table ends the shared allocation, included) all run big members at the same time"""
    return [(i // G) % 2 for i in range(N)]


@pytest.mark.gpu
@pytest.mark.parametrize("case", list(SAVEAT_CASES))
def test_member_loop_reuses_scratch_bitwise(probe, case):
    """N = 3 (grid x 4) + 1 members on a 2-block grid, ~3000-segment and few-segment integrands alternating in every warp,
    each scaled by its own factor: every member's result is bitwise equal to that member integrated alone, its segment
    count is the restatement's over the data intervals (in the loop's order), and its integral the exact one.  K = 0: the
    big members fill the partial last block of keys (index >= 3072), the guard after the block's tables stays intact, and
    every warp's block maxima sit at the stride quad_smem sizes and equal the maxima of its keys bit for bit."""
    grid, t0, t1 = 2, -1.0, 3.0
    G = grid * 4
    saveat = np.array(SAVEAT_CASES[case], dtype=np.float64)
    sets = [make_steps(*ML_BIG, 3), ML_SMALL]
    N = 3 * G + 1
    which = _member_kinds(N, G)
    for g in range(G):                                 # test construction: every warp runs big, then small, then big
        assert [which[i] for i in range(g, N, G)][:3] == [0, 1, 0]
    mult = np.array([1.0 + 0.125 * i for i in range(N)])
    dp, calls, g, l1_bad = _member_loop(probe, sets, which, mult, saveat, t0, t1, 0.0, ML_RTOL, ML_MAXSEG, grid)
    assert g.all(), "store past the block-maxima tables"
    refs = []
    for jt, js in sets:
        parts = [quadgk_ref(step_fn(jt, js), 3, lo, hi, 0.0, ML_RTOL, ML_MAXSEG, jt) for lo, hi in _intervals(saveat, t0, t1)]
        assert all(p["ok"] and p["margin"] > 1e-9 and p["near"] > 8 for p in parts), "test construction"
        refs.append(parts)
    if case == "K0":
        assert 32 * (ML_MAXSEG // 32) < refs[0][0]["nseg"] <= ML_MAXSEG, f"test construction: {refs[0][0]['nseg']} segments"
        assert l1_bad == 0, f"{l1_bad} block maxima are not where quad_smem puts the warp's table, or not the maxima of its keys"
    for i in range(N):
        alone, calls1 = _member_loop(probe, [sets[which[i]]], [0], mult[i:i + 1], saveat, t0, t1, 0.0, ML_RTOL, ML_MAXSEG, 1)[:2]
        assert np.array_equal(dp[:, i], alone[:, 0]), f"member {i}: {dp[:, i]} vs alone {alone[:, 0]}"
        parts = refs[which[i]]
        assert calls[i] == calls1[0] == sum(p["nseg"] for p in parts), f"member {i}: {calls[i]} / {calls1[0]} segments"
        ref = mult[i] * sum(p["I"] for p in parts)
        assert np.abs(dp[:, i] - ref).max() <= 1e-13 * np.abs(ref).max()
        jt, js = sets[which[i]]
        exact = np.array(step_exact(jt, js, t0, t1, Fraction(mult[i])))
        tol = ML_RTOL * mult[i] * sum(np.linalg.norm(p["I"]) for p in parts)       # jumps hidden next to a segment end: see _compare
        assert np.abs(dp[:, i] - exact).max() <= max(tol, np.abs(ref - exact).max()) + 1e-13 * np.abs(ref).max()


# ------------------------------------------------------------------------------------------------------------------------
# the production integrand contexts on synthetic records


D, PQ = 2, 3
ROS_D = 0.29289321881345247559915563789515
IC = 1.0 / (1 - 2 * ROS_D)


def _pad4(n):
    return (n + 3) // 4 * 4


class Records:
    """Member-major dense solutions of one member: forward knots ftT[nf + 1] with records, reverse ends rend[nrev] (descending)
    with records, built continuous (each record starts where the previous interpolant ends) so that the integrand is a
    continuous piecewise polynomial.  kind 0: Rosenbrock23 layouts, 1: adaptive Tsit5 layouts."""

    def __init__(self, kind, fknots, rends, t1, seed, amp=0.05):
        rng = np.random.default_rng(seed)
        self.kind = kind
        self.ftT = np.asarray(fknots, np.float64)
        self.nf = len(self.ftT) - 1
        self.rend = np.asarray(rends, np.float64)
        self.nrev = len(self.rend)
        self.R = 0.3 * rng.standard_normal((7, 4))
        self.B = rng.standard_normal((PQ, D, D))
        nk = 2 if kind == 0 else 4          # forward: Ros k1, k2; T5a c0..c3
        FWP = _pad4(3 * D + 3) if kind == 0 else 8 * D + 4
        self.fk = amp * rng.standard_normal((self.nf, nk, D))
        self.fu = np.zeros((self.nf, D))
        u = np.array([1.0, -0.5])
        self.frecT = np.zeros((self.nf + (kind == 1), FWP))
        for i in range(self.nf):
            ta, h = self.ftT[i], self.ftT[i + 1] - self.ftT[i]
            self.fu[i] = u
            r = self.frecT[i]
            r[:D] = u
            r[D:D + nk * D] = self.fk[i].ravel()
            base = 3 * D if kind == 0 else 8 * D
            r[base], r[base + 1] = ta, h
            with np.errstate(divide="ignore"):
                r[base + 2] = 1.0 / h
            u = self._y(i, np.array([1.0]), np.array([h]))[0] if h != 0 else u
        nkr = 2 if kind == 0 else 7
        RWP = _pad4(3 + 3 * D) if kind == 0 else _pad4(3 + 8 * D)
        self.rk = amp * rng.standard_normal((self.nrev, nkr, D))
        self.rz = np.zeros((self.nrev, D))
        self.rts = np.concatenate([[t1], self.rend[:-1]])
        self.rh = self.rend - self.rts
        self.rrec = np.zeros((self.nrev, RWP))
        z = np.array([0.3, 0.8])
        for j in range(self.nrev):
            self.rz[j] = z
            r = self.rrec[j]
            r[0], r[1] = self.rts[j], self.rh[j]
            r[2:2 + D] = z
            r[2 + D:2 + D + nkr * D] = self.rk[j].ravel()
            with np.errstate(divide="ignore"):
                r[2 + (1 + nkr) * D] = 1.0 / self.rh[j]
            if self.rh[j] != 0:
                z = self._lam(j, np.array([1.0]))[0]

    def _y(self, i, th, h):
        u, k = self.fu[i], self.fk[i]
        if self.kind == 0:
            c1, c2 = th * (1 - th) * IC, th * (th - 2 * ROS_D) * IC
            return u + h[:, None] * (c1[:, None] * k[0] + c2[:, None] * k[1])
        g = (h * th)[:, None]
        return u + g * (k[0] + th[:, None] * (k[1] + th[:, None] * (k[2] + th[:, None] * k[3])))

    def _lam(self, j, th):
        z, k, h = self.rz[j], self.rk[j], self.rh[j]
        if self.kind == 0:
            c1, c2 = th * (1 - th) * IC, th * (th - 2 * ROS_D) * IC
            return z + h * (c1[:, None] * k[0] + c2[:, None] * k[1])
        w = th[:, None] * (self.R[:, 0] + th[:, None] * (self.R[:, 1] + th[:, None] * (self.R[:, 2] + th[:, None] * self.R[:, 3])))
        return z + h * (w @ k)

    def integrand(self, t):
        """the context's integrand at points t inside pieces (on no knot)"""
        iv = np.searchsorted(self.ftT[1:self.nf], t, side="left")          # interior forward knots < t
        lo = np.searchsorted(-self.rend[:self.nrev - 1], -t, side="left")   # reverse ends > t
        y, lam = np.zeros((len(t), D)), np.zeros((len(t), D))
        for i in np.unique(iv):
            m = iv == i
            h = self.ftT[i + 1] - self.ftT[i]
            y[m] = self._y(i, (t[m] - self.ftT[i]) / h, np.full(m.sum(), h))
        for j in np.unique(lo):
            m = lo == j
            lam[m] = self._lam(j, (t[m] - self.rts[j]) / self.rh[j])
        return np.einsum("qjk,nj,nk->nq", self.B, y, lam)

    def exact(self, a, b):
        """piecewise 8-point Gauss-Legendre (exact for these degree <= 8 pieces up to rounding), fsum over the pieces"""
        cuts = np.unique(np.concatenate([[a, b], self.ftT[(self.ftT > a) & (self.ftT < b)], self.rend[(self.rend > a) & (self.rend < b)]]))
        lo, hi = cuts[:-1], cuts[1:]
        x, wt = np.polynomial.legendre.leggauss(8)
        t = (0.5 * (lo + hi))[:, None] + (0.5 * (hi - lo))[:, None] * x[None, :]
        v = self.integrand(t.ravel()).reshape(len(lo), 8, PQ)
        contrib = (0.5 * (hi - lo))[:, None] * np.einsum("k,nkq->nq", wt, v)
        return np.array([math.fsum(contrib[:, q]) for q in range(PQ)])


def _run_ctx(probe, rec, a, b, atol, rtol, maxseg):
    import torch
    ts = [_dev(rec.ftT), _dev(rec.frecT.ravel()), _dev(rec.rrec.ravel()), _dev(rec.rend)]
    out = torch.full((PQ,), float("nan"), dtype=torch.float64, device="cuda")
    info = torch.full((3,), -1, dtype=torch.int32, device="cuda")
    bad = torch.full((2,), 12345, dtype=torch.int32, device="cuda")
    B = np.ascontiguousarray(rec.B, np.float64); R = np.ascontiguousarray(rec.R, np.float64)
    _check(probe.probe_ctx(rec.kind, B.ctypes.data, R.ctypes.data, *[x.data_ptr() for x in ts], rec.nf, rec.nrev, a, b, atol, rtol, maxseg,
                           out.data_ptr(), info.data_ptr(), bad.data_ptr()))
    ok, n, guard = (int(x) for x in info.cpu().numpy())
    return out.cpu().numpy(), ok, n, guard, bad.cpu().numpy()


def _ctx_layout(case):
    rng = np.random.default_rng({"geometric": 1, "dyadic": 2, "zero_length": 3}[case])
    if case == "geometric":           # 5000 forward knots geometric over 1e-8 .. 1e2, reverse ends on another ratio
        a, b = 0.0, 100.0
        f = np.concatenate([[0.0], np.geomspace(1e-8, 100.0, 5000)])
        r = np.concatenate([np.geomspace(3e-8, 100.0, 3001)[:-1][::-1], [0.0]])
    elif case == "dyadic":            # knots exactly on bisection points of the data interval
        a, b = 0.0, 1.0
        f = np.unique(np.concatenate([np.arange(65) / 64.0, rng.uniform(0, 1, 40)]))
        r = np.unique(np.concatenate([np.arange(129) / 128.0, rng.uniform(0, 1, 30)]))[::-1].copy()
    else:                             # zero-length steps (h = 0) in both solutions
        a, b = 0.0, 1.0
        f = np.sort(np.concatenate([np.linspace(0, 1, 300), np.linspace(0, 1, 300)[10::37], [0.5, 0.5]]))
        r = np.sort(np.concatenate([np.linspace(0, 1, 200), np.linspace(0, 1, 200)[5::23]]))[::-1].copy()
    return a, b, f, r


# rtol per layout: the geometric one (8000 knots) needs ~15 000 segments at 1e-10
CTX_RTOL = {"geometric": 1e-8, "dyadic": 1e-10, "zero_length": 1e-10}


@pytest.mark.gpu
@pytest.mark.parametrize("kind", [0, 1], ids=["ros", "t5a"])
@pytest.mark.parametrize("case", ["geometric", "dyadic", "zero_length"])
def test_production_context_lookups_and_integral(probe, kind, case):
    """Every lookup of the production context agrees with a scan over all knots and lies inside the segment's brackets;
    the integral matches the exact piecewise integral to 2 rtol |I| (the restatement on these kinked integrands lands at
    up to 1.06 rtol |I|: the error estimate is not a bound)."""
    a, b, f, r = _ctx_layout(case)
    rec = Records(kind, f, r, b, seed=40 + kind)
    atol, rtol, maxseg = 0.0, CTX_RTOL[case], 16384
    I, ok, n, guard, bad = _run_ctx(probe, rec, a, b, atol, rtol, maxseg)
    assert ok and guard
    assert bad[0] == 0, f"{bad[0]} lookups disagree with the scan over all knots ({n} segments)"
    assert bad[1] == 0, f"{bad[1]} lookups fall outside the segment's bracket"
    exact = rec.exact(a, b)
    assert np.abs(I - exact).max() <= 2 * max(atol, rtol * np.linalg.norm(exact)), (I, exact, n)
    print(f"{case} {['ros', 't5a'][kind]}: {n} segments, |I - exact| / |I| = {np.abs(I - exact).max() / np.linalg.norm(exact):.2e}")
