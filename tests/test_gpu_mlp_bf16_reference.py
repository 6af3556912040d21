"""The bf16 tensor-core neural-ODE kernels (csrc/mlp_tc.cuh, 32 members per CTA; csrc/mlp_tc_wide.cuh, 128 members per
CTA; dtype = "bf16_f32acc") through the public DeviceEnsemble API against the bf16 twin of tests/mlp_bf16_twin.py, run
with the device's own tanh.approx.f32 (tests/csrc/wgmma_probe.cu: probe_tanh_approx).

Every group runs both layouts: the host takes the narrow one while ceil(N / 32) <= 2 n_SM.  Large ensembles repeat a
prime number K of distinct states (member m starts at base[m % K], and carries the cotangent of base member m % K); a
member's result is bit-identical wherever it sits (test_gpu_parity_mlp.test_mlp_bf16_member_permutation), so the twin
runs K members, weighs each by its count for dp, and every member of the kernel is compared.

The twin reproduces the bf16 roundings, the fp32 arithmetic in the kernels' order and tanh.approx.f32 exactly.  What is
left is the accumulation order inside wgmma.  Each comparison's bound is derived, never tuned (mlp_bf16_twin.derive):
gamma_n sum |terms| of the gradient GEMMs' fp32 chains, plus 4x the spread of the twin when every member-GEMM result
moves at random within gamma_64 sum |terms|.  Every case prints observed / bound, and the bounds relative to scale.

* Device helpers: pack_bf16 against the twin's rounding bit for bit; tanh.approx.f32 within its 2^-11 relative error.
* Every checkpoint: saved at every grid point; from the kernel's own saved[n], one twin step gives saved[n + 1]
  (a failure names the step); the whole trajectory against the free-running twin.
* One-step reverse windows: T = dt, one member per kernel checkpoint, an explicit cotangent at t_{n+1}; du0 of member n
  is the reverse map of step n (a failure names the step); dp of single-member windows.
* Whole gradients, pairwise over sensealg x {scalar, per-component, explicit} cost x {plain, no_start, set_reverse} x
  dt in {0.05, 0.25} x N in {1, 33, 64 n_SM, 64 n_SM + 1, 64 n_SM + 127}, and C4 itself (4096 members, dt = 0.05,
  30 saves).  The forward saves every grid point, and the twin's reverse pass runs over the kernel's own checkpoints,
  as the kernel's does: a bf16 rounding flipped early in a free-running forward pass would otherwise move every later
  state by ~1e-3 and hide the reverse pass under it.
* Saturation: |u0| up to 6, first-layer features at bf16 H1 = +-1 (1 - H1^2 = 0).
* Exact relation: an explicit cotangent times 2^k, k in {-60, +40}, scales du0 and dp by exactly 2^k.
"""
import ctypes as C
import itertools
import os
import sys
import time

import numpy as np
import pytest

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(HERE)
for d in (ROOT, HERE):
    if d not in sys.path:
        sys.path.insert(0, d)

import mlp_bf16_twin as T
import mlp_restatement as R
import test_mlp_restatement as TM
from test_gpu_wgmma_probe import probe, probe_so  # noqa: F401  (the fixtures that build and load tests/csrc/wgmma_probe.cu)

pytestmark = pytest.mark.gpu
LAYOUTS = ("narrow", "wide")
DT_END = TM.T_END

# The ceilings of the derived bounds, relative to each output's scale: 1e-3 wherever the derivation reaches it (one twin
# step from a kernel checkpoint, du0 of one-step windows).  Where it does not, the ceiling is stated here, and the term
# that dominates is in every case the perturbation term (4x the spread), not gamma_n sum |terms|: a member-GEMM result
# moved within the measured wgmma residual (T.WGMMA_RESIDUAL) now and then flips the bf16 rounding of an H1 / dZ2 / dZ1
# entry it feeds, a 2^-8 relative step of one term.  On an H100 the derived bounds reach 6e-3 of scale over a
# free-running trajectory, 2e-2 over a whole gradient (dt = 0.25, and small dp blocks of explicit-cost cases), 7e-3 at the
# saturation edge and 6e-2 for one dp block of a single-member one-step window.  The kernels stay at or below 0.35 of
# every bound; the sharp checks of the Gauss-node gradient are the window gradients (bounds 1e-6 .. 1e-4 at dt = 0.05).
CEILINGS = {"step": T.CEILING, "window": T.CEILING, "window_dp": 1e-1, "trajectory": 1e-2, "whole": 3e-2, "saturation": 1e-2}


def _nsm():
    import torch
    return torch.cuda.get_device_properties(0).multi_processor_count


def _layout(N):
    return "narrow" if -(-N // 32) <= 2 * _nsm() else "wide"


@pytest.fixture(scope="module")
def dev(probe_so):  # noqa: F811
    lib = C.CDLL(probe_so)
    lib.probe_tanh_approx.argtypes = [C.c_void_p, C.c_void_p, C.c_int64]
    lib.probe_pack_bf16.argtypes = [C.c_void_p, C.c_void_p, C.c_int64]
    lib.probe_tanh_approx.restype = lib.probe_pack_bf16.restype = C.c_int
    return lib


@pytest.fixture(scope="module")
def tanh_dev(dev):
    """tanh.approx.f32 of the device, element-wise, on an array of fp32 values"""
    import torch

    def f(x):
        x = np.asarray(x, dtype=np.float32)
        xd = torch.from_numpy(np.ascontiguousarray(x)).cuda()
        yd = torch.empty_like(xd)
        assert dev.probe_tanh_approx(xd.data_ptr(), yd.data_ptr(), xd.numel()) == 0
        return yd.cpu().numpy().astype(np.float64)
    return f


def _engine(sa, N, saveat, dt, T_, cost, no_start=False):
    import scimlsensitivity_jl_b200 as b
    c = TM.COSTS[cost]
    return b.DeviceEnsemble("mlp", sa, "tsit5_fixed", N, saveat, (0.0, T_), dt, dtype="bf16_f32acc", no_start=no_start,
                            cost=None if cost == "explicit" else b.AffineCost(*c))


def _cyclic(N, K, seed, amp=2.0):
    base = T.f32(np.random.default_rng(seed).uniform(-amp, amp, (2, K)))
    idx = np.arange(N) % K
    return base[:, idx], base, np.bincount(idx, minlength=K), idx


def _report(tag, group, rat, ceil):
    line = f"{tag}: observed/bound " + " ".join(f"{k} {v:.2f}" for k, v in rat.items()) + " | bound/scale " + \
        " ".join(f"{k} {v:.1e}" for k, v in ceil.items())
    print(line)
    assert max(ceil.values()) <= CEILINGS[group], line
    assert max(rat.values()) <= 1.0, line


# ------------------------------------------------------------------------------------------------------------------------
# device helpers


def test_pack_bf16_matches_the_twin_bit_for_bit(dev):
    import torch
    rng = np.random.default_rng(3)
    ties = (np.arange(0, 1 << 16, dtype=np.uint32) << 16) | 0x8000
    pw = np.exp2(np.arange(-149, 128, dtype=np.float64)).astype(np.float32)
    x = np.concatenate([ties.view(np.float32), rng.integers(0, 1 << 32, 100000, dtype=np.uint64).astype(np.uint32).view(np.float32),
                        np.nextafter(pw, np.float32(0)), pw, np.nextafter(pw, np.float32(np.inf)),
                        (np.arange(1, 4096, dtype=np.uint32) * 2039).view(np.float32)])
    x = np.concatenate([x, -x])
    x = x[np.isfinite(x)]
    x = x[: x.size // 2 * 2]
    xd = torch.from_numpy(x).cuda()
    out = torch.empty(x.size // 2, dtype=torch.int32, device="cuda")
    assert dev.probe_pack_bf16(xd.data_ptr(), out.data_ptr(), x.size // 2) == 0
    w = out.cpu().numpy().view(np.uint32)
    got = np.empty(x.size, dtype=np.uint32)
    got[0::2], got[1::2] = w << 16, w & 0xFFFF0000                  # the first of a pair in the low half
    ref = np.asarray(T.bf16(x), dtype=np.float32).view(np.uint32)
    bad = np.flatnonzero(got != ref)
    assert bad.size == 0, [(hex(x.view(np.uint32)[i]), hex(got[i]), hex(ref[i])) for i in bad[:10]]


def test_tanh_approx_is_within_its_documented_error(tanh_dev):
    x = np.concatenate([np.linspace(-10, 10, 200001), np.exp2(np.arange(-30, 4.0, 0.25))]).astype(np.float32)
    x = np.concatenate([x, -x])
    ref = np.tanh(x.astype(np.float64))
    err = np.abs(tanh_dev(x) - ref) / np.maximum(np.abs(ref), 1e-30)
    print(f"tanh.approx.f32: largest relative error {err.max():.2e} (2^{np.log2(err.max()):.2f})")
    assert err.max() <= 2.0 ** -10.9


def _member_gemm_residual(probe, layout, tile, seed):
    """|wgmma - exact| / (2^-24 sum |terms|) over one member GEMM of realistic operands: forward (tile TB = bf16 H1 in
    (-1, 1), B = bf16 W2) or backward (tile TA = bf16 wt dZ2 of mixed signs and magnitudes, B = bf16 W2'); the exact sum
    is the fp64 one (64 products of 8-bit significands: exact in fp64)"""
    import torch
    rng = np.random.default_rng(seed)
    rows = 64 if layout == "narrow" else 128
    F = 80 if tile == "TB" else 128
    A = np.zeros((rows, F))
    if tile == "TB":
        A[:, :64] = T.bf16(np.tanh(rng.standard_normal((rows, 64)) * 2.0))
    else:
        A[:, :64] = T.bf16(rng.standard_normal((rows, 64)) * np.exp2(rng.integers(-12, 1, (rows, 64))))
    p = T.f32(R.weights(seed))
    W2 = T.bf16(R.unpack(p)[2])
    B = W2.T if tile == "TB" else W2                                         # D = A W2' (TB) or A W2 (TA)
    members = 32 if layout == "narrow" else 128
    D = torch.full((members, 64), float("nan"), dtype=torch.float32, device="cuda")
    keep = [torch.tensor(p, dtype=torch.float32, device="cuda"), torch.tensor(A, dtype=torch.float32, device="cuda")]
    assert probe.probe_member_gemm(1 if layout == "wide" else 0, F, keep[0].data_ptr(), keep[1].data_ptr(),
                                   0 if tile == "TB" else 1, D.data_ptr()) == 0
    got = D.cpu().numpy().astype(np.float64)
    exact = (A[:, :64] @ B)[:members]
    sabs = (np.abs(A[:, :64]) @ np.abs(B))[:members]
    ok = sabs > 0
    return np.abs(got - exact)[ok] / (T.EPS32 * sabs[ok]), got[ok] == T.f32(exact[ok])


@pytest.mark.parametrize("tile", ["TB", "TA"])
@pytest.mark.parametrize("layout", LAYOUTS)
def test_member_gemm_residual_is_within_the_twins_model(probe, layout, tile):  # noqa: F811
    """The twin moves each member-GEMM result within T.WGMMA_RESIDUAL x 2^-24 sum |terms| (mlp_bf16_twin): the largest
    deviation of wgmma from the exact sum measured here over 20 GEMMs of realistic operands per layout and tile must stay
    within it."""
    r, same = zip(*(_member_gemm_residual(probe, layout, tile, seed) for seed in range(1, 21)))
    r, same = np.concatenate(r), np.concatenate(same)
    print(f"{layout} {tile}: wgmma - exact, largest {r.max():.3f} x 2^-24 sum|terms| (mean {r.mean():.3f}); "
          f"{same.mean():.4f} of the entries equal the correctly rounded sum")
    assert r.max() <= T.WGMMA_RESIDUAL, r.max()


# ------------------------------------------------------------------------------------------------------------------------
# every checkpoint


def _forward_case(layout, seed=12, amp=2.0, dt=0.05):
    S = int(round(DT_END / dt))
    if layout == "narrow":
        N, K = 40, 40
    else:
        N, K = 64 * _nsm() + 1, 37
    u0, base, cnt, idx = _cyclic(N, K, seed, amp)
    assert _layout(N) == layout
    return N, K, S, dt, u0, base, cnt, idx


@pytest.mark.parametrize("layout", LAYOUTS)
def test_every_checkpoint(layout, tanh_dev):
    N, K, S, dt, u0, base, cnt, idx = _forward_case(layout)
    p = T.f32(R.weights())
    eng = _engine("interpolating", N, np.arange(S + 1) * dt, dt, DT_END, "scalar")
    saved, status = eng.forward(u0, p)
    eng.close()
    assert (np.asarray(status) == 0).all()
    saved = np.asarray(saved, dtype=np.float64)
    assert np.array_equal(saved[0], u0)
    kern = saved[:, :, :K]                                                    # [S+1][2][K]: members 0..K-1 = base
    assert np.array_equal(saved, kern[:, :, idx])                             # every copy of a state: the same bits
    # one twin step from each of the kernel's own checkpoints
    starts = kern[:-1].transpose(1, 0, 2).reshape(2, S * K)
    step = lambda perturb: {"us": T.Twin(p, dt, tanh=tanh_dev, layout=layout, perturb=perturb).forward(starts, 1)[0]}
    b1, bd1 = T.derive(step)
    got = kern[1:].transpose(1, 0, 2).reshape(2, S * K)
    err = (np.abs(got - b1["us"][1]) / T.member_scale(b1["us"][1])).reshape(2, S, K).max(axis=(0, 2))
    print(f"{layout}: one twin step from every kernel checkpoint, worst step {int(err.argmax())}, largest error {err.max():.1e}, "
          f"{int((err == 0).sum())} of {S} steps bit-identical for all members")
    bad = [(n, float(e)) for n, e in enumerate(err) if e > bd1["us"]]
    assert not bad, f"steps over the bound {bd1['us']:.1e}: {bad}"
    _report(f"{layout} step by step", "step", T.ratios({"us": got[None]}, {"us": b1["us"][1:]}, bd1), {"us": bd1["us"]})
    # the whole trajectory against the free-running twin
    run = lambda perturb: {"us": T.Twin(p, dt, tanh=tanh_dev, layout=layout, perturb=perturb).forward(base, S)[0]}
    b2, bd2 = T.derive(run)
    _report(f"{layout} trajectory", "trajectory", T.ratios({"us": kern}, b2, bd2), T.ceilings(b2, bd2))


# ------------------------------------------------------------------------------------------------------------------------
# one-step reverse windows


@pytest.mark.parametrize("sa", ["interpolating", "gauss"])
@pytest.mark.parametrize("layout", LAYOUTS)
def test_one_step_windows(layout, sa, tanh_dev):
    """T = dt = 0.05: member n starts at the kernel's checkpoint u_n of a 31-step trajectory and carries an explicit
    cotangent at t_{n+1}; du0 of member n is the reverse map of step n.  Then single-member windows give that step's dp."""
    dt, S = 0.05, 31
    p = T.f32(R.weights())
    rng = np.random.default_rng(30)
    u0 = T.f32(rng.uniform(-2, 2, (2, 1)))
    eng = _engine(sa, 1, np.arange(S + 1) * dt, dt, S * dt, "scalar")
    traj = np.asarray(eng.forward(u0, p)[0], dtype=np.float64)[:S, :, 0]      # the kernel's u_0 .. u_{S-1}
    eng.close()
    starts = traj.T                                                           # [2][S]: one window per member
    dLdu = T.f32(rng.standard_normal((1, 2, S)))
    N = S if layout == "narrow" else 64 * _nsm() + 1
    idx = np.arange(N) % S
    assert _layout(N) == layout

    def window(cols, n_dev):
        ix = np.arange(n_dev) % len(cols)
        eng = _engine(sa, n_dev, np.array([dt]), dt, dt, "explicit")
        eng.forward(starts[:, cols][:, ix], p)
        du0, dp = (np.asarray(x, dtype=np.float64) for x in eng.reverse(dLdu[:, :, cols][:, :, ix]))
        eng.close()
        cnt = np.bincount(ix, minlength=len(cols))
        runner = lambda perturb: T.run(p, starts[:, cols], dt, 1, {1: 0}, "explicit", dLdu[:, :, cols], sensealg=sa, cnt=cnt,
                                       tanh=tanh_dev, layout=_layout(n_dev), perturb=perturb)
        base, bounds = T.derive(runner)
        return du0, dp, base, bounds, ix

    du0, _, base, bounds, ix = window(list(range(S)), N)
    err = (np.abs(du0 - base["du0"][:, ix]) / T.member_scale(base["du0"][:, ix])).max(axis=0)
    per_step = np.zeros(S)
    np.maximum.at(per_step, ix, err)
    print(f"{layout} {sa}: one-step windows, largest du0 error {err.max():.1e} at step {int(per_step.argmax())}, "
          f"{int((per_step == 0).sum())} of {S} steps bit-identical")
    bad = [(n, float(e)) for n, e in enumerate(per_step) if e > bounds["du0"]]
    assert not bad, f"steps over the bound {bounds['du0']:.1e}: {bad}"
    _report(f"{layout} {sa} windows du0", "window", T.ratios({"du0": du0}, base, bounds, cols=ix), {"du0": bounds["du0"]})
    if layout == "narrow":
        for n in (0, 2, S - 1):
            _, dp, base, bounds, _ = window([n], 1)
            _report(f"{sa} window {n} dp", "window_dp", T.ratios({"dp": dp}, base, bounds),
                    {k: v for k, v in T.ceilings(base, bounds).items() if k in R.BLOCKS})


WINDOW_K = 7            # windows (distinct members) of test_gauss_window_gradients: steps 0 .. 6 of one trajectory


def window_inputs(dt, seed=31):
    """-> (p, u0 [2][1], dLdu [1][2][WINDOW_K]) of test_gauss_window_gradients"""
    rng = np.random.default_rng(seed)
    return T.f32(R.weights()), T.f32(rng.uniform(-2, 2, (2, 1))), T.f32(rng.standard_normal((1, 2, WINDOW_K)))


def window_runner(p, starts, dt, dLdu, cnt=None, **kw):
    """the twin of test_gauss_window_gradients: one GaussAdjoint step from each start, explicit cotangent at t + dt"""
    return lambda perturb: T.run(p, starts, dt, 1, {1: 0}, "explicit", dLdu, sensealg="gauss", cnt=cnt, perturb=perturb, **kw)


@pytest.mark.parametrize("dt", [0.05, 0.25])
@pytest.mark.parametrize("layout", LAYOUTS)
def test_gauss_window_gradients(layout, dt, tanh_dev):
    """GaussAdjoint one-step windows, both layouts: members start at the kernel's checkpoints u_0 .. u_6 of one trajectory
    (wide: 64 n_SM + 1 members cycling through them) with an explicit cotangent at t_{n+1}.  dp here is the sum over the
    windows of the Gauss-node gradient of one step, which is where the Gauss-node lambda and y (ka[6], the node order, k7)
    enter; du0 per member as in test_one_step_windows."""
    p, u0, dLdu = window_inputs(dt)
    eng = _engine("gauss", 1, np.arange(WINDOW_K + 1) * dt, dt, WINDOW_K * dt, "scalar")
    starts = np.asarray(eng.forward(u0, p)[0], dtype=np.float64)[:WINDOW_K, :, 0].T        # the kernel's u_0 .. u_6
    eng.close()
    N = WINDOW_K if layout == "narrow" else 64 * _nsm() + 1
    ix = np.arange(N) % WINDOW_K
    assert _layout(N) == layout
    eng = _engine("gauss", N, np.array([dt]), dt, dt, "explicit")
    eng.forward(starts[:, ix], p)
    du0, dp = (np.asarray(x, dtype=np.float64) for x in eng.reverse(dLdu[:, :, ix]))
    eng.close()
    base, bounds = T.derive(window_runner(p, starts, dt, dLdu, np.bincount(ix, minlength=WINDOW_K), tanh=tanh_dev, layout=layout))
    _report(f"{layout} gauss windows dt {dt}", "window_dp", T.ratios({"du0": du0, "dp": dp}, base, bounds, cols=ix),
            T.ceilings(base, bounds))


# ------------------------------------------------------------------------------------------------------------------------
# whole gradients


SIZES = {"1": lambda nsm: 1, "33": lambda nsm: 33, "64nsm": lambda nsm: 64 * nsm, "64nsm+1": lambda nsm: 64 * nsm + 1,
         "64nsm+127": lambda nsm: 64 * nsm + 127}
FACTORS = (("interpolating", "gauss"), ("scalar", "vector", "explicit"), ("plain", "no_start", "set_reverse"), (0.05, 0.25), tuple(SIZES))


def _pairwise(factors):
    """a greedy pairwise cover: rows of the full product added while they cover a not yet covered pair of levels"""
    need = {(i, a, j, b) for i, j in itertools.combinations(range(len(factors)), 2) for a in factors[i] for b in factors[j]}
    rows = []
    cands = list(itertools.product(*factors))
    while need:
        gain = lambda r: sum((i, r[i], j, r[j]) in need for i, j in itertools.combinations(range(len(r)), 2))
        best = max(cands, key=gain)
        rows.append(best)
        need -= {(i, best[i], j, best[j]) for i, j in itertools.combinations(range(len(best)), 2)}
    return rows


WHOLE = _pairwise(FACTORS)


def _whole_label(c):
    return f"{c[0]}-{c[1]}-{c[2]}-dt{c[3]}-N{c[4]}"


def whole_inputs(sa, cost, mode, dt, size, nsm, seed=3):
    """the inputs of one whole-gradient case -> dict(N, K, S, grid, u0, base, cnt, idx, p, sos, rev_t, dL [K saves][2][K])"""
    N = SIZES[size](nsm)
    K = min(N, 37)
    S = int(round(DT_END / dt))
    grid = np.arange(S + 1) * dt
    u0, base, cnt, idx = _cyclic(N, K, seed)
    rev_t = grid[1::3] if mode == "set_reverse" else None
    sos = {int(round(t / dt)): k for k, t in enumerate(rev_t)} if mode == "set_reverse" else {n: n for n in range(S + 1)}
    dL = T.f32(np.random.default_rng(seed + 100).standard_normal((len(sos), 2, K))) if cost == "explicit" else None
    return dict(N=N, K=K, S=S, grid=grid, u0=u0, base=base, cnt=cnt, idx=idx, p=T.f32(R.weights()), sos=sos, rev_t=rev_t, dL=dL)


def whole_runner(c, w, us=None, **kw):
    """the twin of one whole-gradient case c = (sa, cost, mode, dt, size) with inputs w"""
    sa, cost, mode, dt, _ = c
    return lambda perturb: T.run(w["p"], w["base"], dt, w["S"], w["sos"], TM.COSTS[cost], w["dL"], sensealg=sa,
                                 no_start=mode == "no_start", cnt=w["cnt"], us=us, perturb=perturb, **kw)


def _whole_case(sa, cost, mode, dt, size, tanh):
    import scimlsensitivity_jl_b200 as b
    c = (sa, cost, mode, dt, size)
    w = whole_inputs(*c, _nsm())
    other = "gauss" if sa == "interpolating" else "interpolating"
    eng = _engine(other if mode == "set_reverse" else sa, w["N"], w["grid"], dt, DT_END, cost, no_start=mode == "no_start")
    saved, status = eng.forward(w["u0"], w["p"])
    assert (np.asarray(status) == 0).all()
    if mode == "set_reverse":
        eng.set_reverse(sa, cost=None if cost == "explicit" else b.AffineCost(*TM.COSTS[cost]), t=w["rev_t"])
    du0, dp = (np.asarray(x, dtype=np.float64) for x in eng.reverse(None if w["dL"] is None else w["dL"][:, :, w["idx"]]))
    eng.close()
    us = np.asarray(saved, dtype=np.float64)[:, :, :w["K"]]
    tb, bounds = T.derive(whole_runner(c, w, us=us, tanh=tanh, layout=_layout(w["N"])))
    return du0, dp, tb, bounds, w["idx"]


@pytest.mark.parametrize("c", WHOLE, ids=_whole_label)
def test_whole_gradient(c, tanh_dev):
    t0 = time.perf_counter()
    du0, dp, base, bounds, idx = _whole_case(*c, tanh=tanh_dev)
    _report(f"{_whole_label(c)} ({_layout(SIZES[c[4]](_nsm()))}, {time.perf_counter() - t0:.1f} s)", "whole",
            T.ratios({"du0": du0, "dp": dp}, base, bounds, cols=idx), T.ceilings(base, bounds))


@pytest.mark.parametrize("sa", ["interpolating", "gauss"])
def test_c4_at_production_size(sa, tanh_dev):
    """BASELINE C4: 4096 members, dt = 0.05, saveat = 0.05 .. 1.5 (30 saves), scalar affine cost; 61 distinct states"""
    N, K, dt, S = 4096, 61, 0.05, 30
    saveat = np.linspace(0.05, DT_END, 30)
    u0, base, cnt, idx = _cyclic(N, K, 61)
    p = T.f32(R.weights())
    eng = _engine(sa, N, saveat, dt, DT_END, "scalar")
    saved, _ = eng.forward(u0, p)
    du0, dp = (np.asarray(x, dtype=np.float64) for x in eng.reverse())
    eng.close()
    us = np.concatenate([base[None], np.asarray(saved, dtype=np.float64)[:, :, :K]])
    runner = lambda perturb: T.run(p, base, dt, S, {n: n - 1 for n in range(1, S + 1)}, TM.COSTS["scalar"], sensealg=sa, cnt=cnt,
                                   us=us, tanh=tanh_dev, layout=_layout(N), perturb=perturb)
    tb, bounds = T.derive(runner)
    _report(f"C4 {sa} ({_layout(N)})", "whole", T.ratios({"du0": du0, "dp": dp}, tb, bounds, cols=idx), T.ceilings(tb, bounds))


# ------------------------------------------------------------------------------------------------------------------------
# saturation edge


@pytest.mark.parametrize("layout", LAYOUTS)
def test_saturation_edge(layout, tanh_dev):
    """|u0| up to 6 (two members at (+-6, -+6)): first-layer features saturate, the bf16 H1 is exactly +-1 and 1 - H1^2 = 0;
    the twin must follow the kernel there.  The distance of both from the fp64 restatement is printed (information)."""
    N, K, S, dt, u0, base, cnt, idx = _forward_case(layout, seed=50, amp=6.0, dt=0.25)
    base[:, :2] = [[6.0, -6.0], [-6.0, 6.0]]
    u0 = base[:, idx]
    p = T.f32(R.weights())
    tw = T.Twin(p, dt, tanh=tanh_dev, layout=layout)
    H1 = tw.f(base)[1][1]
    assert (np.abs(H1) == 1.0).sum() > 0, "no saturated first-layer feature"
    print(f"{layout}: {int((np.abs(H1) == 1.0).sum())} of {H1.size} first-layer features at bf16 +-1 at t0")
    sos = {n: n for n in range(S + 1)}
    eng = _engine("gauss", N, np.arange(S + 1) * dt, dt, DT_END, "vector")
    saved, _ = eng.forward(u0, p)
    du0, dp = (np.asarray(x, dtype=np.float64) for x in eng.reverse())
    eng.close()
    us = np.asarray(saved, dtype=np.float64)[:, :, :K]
    runner = lambda perturb: T.run(p, base, dt, S, sos, TM.COSTS["vector"], sensealg="gauss", cnt=cnt, us=us, tanh=tanh_dev,
                                   layout=layout, perturb=perturb)
    tb, bounds = T.derive(runner)
    ref = R.restate("ld", R.problem(dt, S, base, p, sos, TM.COSTS["vector"]), "gauss")
    rdp = (ref["mu"] * cnt).sum(1)
    e = lambda x, r: np.abs(x - r).max() / np.abs(r).max()
    print(f"{layout}: from the fp64 restatement: kernel du0 {e(du0, ref['du0'][:, idx]):.1e} dp {e(dp, rdp):.1e}; "
          f"twin du0 {e(tb['du0'][:, idx], ref['du0'][:, idx]):.1e} dp {e(tb['dp'], rdp):.1e}")
    _report(f"{layout} saturation", "saturation", T.ratios({"du0": du0, "dp": dp}, tb, bounds, cols=idx), T.ceilings(tb, bounds))


# ------------------------------------------------------------------------------------------------------------------------
# exact relation


@pytest.mark.parametrize("k", [-60, 40])
@pytest.mark.parametrize("layout", LAYOUTS)
def test_cotangent_scale_is_exact(layout, k):
    """dLdu -> 2^k dLdu: every operation on the cotangent side (the fp64 stage sums, the fp32 products and sums, the bf16
    roundings, the gradient GEMMs, the reduction) commutes with a power-of-two scale while every value stays in the normal
    fp32 range, which holds for these k (|dLdu| ~ 1, |du0|, |dp| within 1e-6 .. 1e3 of it)."""
    N, K, S, dt, u0, base, cnt, idx = _forward_case(layout, seed=60, dt=0.25)
    p = T.f32(R.weights())
    grid = np.arange(S + 1) * dt
    dL = T.f32(np.random.default_rng(61).standard_normal((S + 1, 2, N)))
    eng = _engine("gauss", N, grid, dt, DT_END, "explicit")
    eng.forward(u0, p)
    du0, dp = (np.asarray(x, dtype=np.float64) for x in eng.reverse(dL))
    du0k, dpk = (np.asarray(x, dtype=np.float64) for x in eng.reverse(dL * 2.0 ** k))
    eng.close()
    tiny = np.finfo(np.float32).tiny
    assert np.abs(du0k[du0k != 0]).min() >= tiny and np.abs(dpk[dpk != 0]).min() >= tiny
    assert np.array_equal(du0k, du0 * 2.0 ** k), np.abs(du0k - du0 * 2.0 ** k).max()
    assert np.array_equal(dpk, dp * 2.0 ** k), np.flatnonzero(dpk != dp * 2.0 ** k)[:20]
