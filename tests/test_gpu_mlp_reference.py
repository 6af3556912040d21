"""The CUDA-core neural-ODE kernels (csrc/mlp.cuh, dtype f64 / f32) through the public DeviceEnsemble API against the
long-double restatement of tests/mlp_restatement.py (the fixed-grid Tsit5 restatement of test_gpu_fixed_reference.py
with a hand-written backprop of the network; its own checks are in tests/test_mlp_restatement.py).

* Every checkpoint: saveat on every grid point; F64 at 1e-13 of the member's largest state, F32 at the bound in
  test_every_checkpoint's docstring.
* Whole gradients, F64, at 1e-12: du0 per member and component (floored at 1e-6 of the member's largest), dp per
  parameter floored at 1e-3 of its block's largest (mlp_restatement.DP_FLOOR).  The pairwise matrix of
  tests/test_mlp_restatement.py (sensealg x scalar / per-component affine / explicit cost x plain / no_start / events x
  dt 0.05, 0.25, 0.5), reverse saves moved with set_reverse(t=...), and the events: scales != 1 and distinct per
  component, one of them 0, on consecutive grid points, on save times, at n = 1 and n = S - 1.  The dt = 0.25 / 0.5
  cases pin the sensealg (the separation guards of test_mlp_restatement.py); dt = 0.05 pins the arithmetic.  The CPU
  oracle's distance from the same restatement is printed beside the device's.
* One-step windows: T = dt, one member per checkpoint u_n of a 30-step trajectory, an explicit cost at t_{n+1}; du0 is
  the reverse map of that one step.  A failure names the step.
* Geometry and exact relations: N in {1, 31, 32, 33, 4096 + 17, 64 n_SM + 1}; a cyclic member shift leaves saved and
  du0 bit-identical; dp(33 members) = dp(first 32) + dp(last 1) bit for bit (the block-order fp64 reduction);
  a repeated reverse() is bitwise the same.
* C4 at production size: 4096 members, dt = 0.05, 30 saves, F64.

Large ensembles repeat a prime number of distinct initial states cyclically (member m starts at base[m % K]), so the
restatement runs K members and weighs each by its count for dp; every member's du0 is compared.  A kernel that read
another member's column would read another distinct state, since no offset the kernels use is a multiple of K.
"""
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

import mlp_restatement as R
import test_mlp_restatement as TM

pytestmark = pytest.mark.gpu
EPS32 = 2.0 ** -24


def _nsm():
    import torch
    return torch.cuda.get_device_properties(0).multi_processor_count


def _engine(sa, N, saveat, dt, T, cost, dtype="f64", no_start=False, events=None):
    import scimlsensitivity_jl_b200 as b
    c = TM.COSTS[cost]
    eng = b.DeviceEnsemble("mlp", sa, "tsit5_fixed", N, saveat, (0.0, T), dt, dtype=dtype, no_start=no_start,
                           cost=None if cost == "explicit" else b.AffineCost(*c))
    if events is not None:
        eng.set_events(*events)
    return eng


def _run(eng, u0, p, dLdu=None):
    saved, status = eng.forward(u0, p)
    assert (np.asarray(status) == 0).all()
    du0, dp = eng.reverse(dLdu)
    return np.array(saved, dtype=np.float64), np.array(du0, dtype=np.float64), np.array(dp, dtype=np.float64)


def _f32(x):
    return np.asarray(x, dtype=np.float32).astype(np.float64)


def _report(tag, du0, dp, ref, oracle=None, tol=1e-12):
    e_u = R.rel_err(du0, ref["du0"])
    e_p, per = R.dp_err(dp, ref["mu"].sum(1))
    line = f"{tag}: device du0 {e_u:.1e} dp {e_p:.1e} (worst block {max(per, key=per.get)})"
    if oracle is not None:
        line += f"; oracle du0 {R.rel_err(oracle['du0'], ref['du0']):.1e} dp {R.dp_err(oracle['dp'], ref['mu'].sum(1))[0]:.1e}"
    print(line)
    assert e_u <= tol and e_p <= tol, line


# ------------------------------------------------------------------------------------------------------------------------


@pytest.mark.parametrize("mode", ["plain", "events"])
@pytest.mark.parametrize("dtype", ["f64", "f32"])
def test_every_checkpoint(dtype, mode):
    """saved at every grid point of C4's grid (dt = 0.05, S = 30), 40 members (a ragged second block), against the
    long-double forward from the same (for F32: fp32-rounded) u0 and p.

    F64: 1e-13 of the member's largest |u|.  F32: each step rounds its six stage inputs and its new state to float
    (the stage sums themselves are fp64), <= 2^-24 relative each, and tanhf errs by <= 2 ulp (CUDA Math API), which
    reaches f through |W3| |W2| (about 8 and 8 for this network, both rows normalised by sqrt(64)) as about 1e2 ulp of
    |f|, times h = 0.05: a local error of at most 8 x 2^-24 of the state's scale per step.  30 steps, amplified by at most
    e^{L T} <= 8 over T = 1.5 for this network: 30 x 8 x 8 x 2^-24 = 1.1e-4 of the member's largest |u|."""
    dt, T = 0.05, 1.5
    S = 30
    N = 40
    grid = np.arange(S + 1) * dt
    rng = np.random.default_rng(12)
    u0, p = rng.uniform(-2, 2, (2, N)), R.weights()
    ev = TM.event_table(S) if mode == "events" else None
    dev_ev = None if ev is None else TM.device_events(ev, dt)
    eng = _engine("interpolating", N, grid, dt, T, "scalar", dtype, events=dev_ev)
    saved, _, _ = _run(eng, u0, p)
    eng.close()
    cast = _f32 if dtype == "f32" else (lambda x: x)
    pr = R.problem(dt, S, cast(u0), cast(p), {n: n for n in range(S + 1)}, TM.COSTS["scalar"], events=ev)
    ref = R.restate("ld", pr, "interpolating")["us"]                 # [S+1][2][N]
    scale = np.abs(ref).max(axis=(0, 1))
    err = (np.abs(saved - ref) / scale).max(axis=(1, 2))           # per step
    bound = 1e-13 if dtype == "f64" else 30 * 8 * 8 * EPS32
    print(f"{dtype} {mode}: largest checkpoint error {err.max():.1e} of the member's scale (bound {bound:.1e}), worst step {int(err.argmax())}")
    assert err.max() <= bound, [(n, float(e)) for n, e in enumerate(err) if e > bound]


def _matrix_case(cost, mode, dt, sa, N=40, seed=3):
    pr, saveat, u0, p, dLdu, dev_ev = TM.setup(N, dt, cost, mode, seed=seed)
    T = TM.T_END
    eng = _engine(sa, N, saveat, dt, T, cost, no_start=mode == "no_start", events=dev_ev)
    _, du0, dp = _run(eng, u0, p, dLdu)
    eng.close()
    ref = R.restate("ld", pr, sa)
    orc = TM.oracle_gradient(sa, cost, mode, dt, saveat, u0, p, dLdu, dev_ev)
    return du0, dp, ref, orc


@pytest.mark.parametrize("c", TM.MATRIX, ids=TM.label)
def test_whole_gradient(c):
    t0 = time.perf_counter()
    du0, dp, ref, orc = _matrix_case(*c)
    _report(TM.label(c), du0, dp, ref, orc)
    print(f"{TM.label(c)}: {time.perf_counter() - t0:.1f} s")


@pytest.mark.parametrize("sa", ["interpolating", "gauss"])
def test_reverse_saves_moved_with_set_reverse(sa):
    """forward with saves on every grid point; the reverse pass re-targeted to every third grid point after t0 with a
    per-component affine cost (dt = 0.25, events on)"""
    import scimlsensitivity_jl_b200 as b
    dt, T, N = 0.25, TM.T_END, 40
    pr, saveat, u0, p, _, dev_ev = TM.setup(N, dt, "scalar", "events", seed=8)
    eng = _engine(sa, N, saveat, dt, T, "scalar", events=dev_ev)
    eng.forward(u0, p)
    t_rev = saveat[1::3]
    eng.set_reverse(sa, cost=b.AffineCost(*TM.COSTS["vector"]), t=t_rev)
    du0, dp = (np.array(x, dtype=np.float64) for x in eng.reverse())
    eng.close()
    pr2 = R.problem(dt, pr.S, u0, p, {int(round(t / dt)): k for k, t in enumerate(t_rev)}, TM.COSTS["vector"],
                    events=TM.event_table(pr.S))
    _report(f"set_reverse {sa}", du0, dp, R.restate("ld", pr2, sa))


@pytest.mark.parametrize("dtype", ["f64", "f32"])
@pytest.mark.parametrize("sa", ["interpolating", "gauss"])
def test_one_step_windows(sa, dtype):
    """T = dt = 0.05, saveat = [dt]: member n starts at the restatement's checkpoint u_n of a 30-step trajectory and
    carries an explicit cotangent at t_{n+1}; du0 of member n is the reverse map of step n.  F64: 1e-14; F32 at
    2000 eps32 (the fixed-step reference's fp32 bound).  Then single-member windows (steps 0, 2 and 29) must give that
    step's dp."""
    dt, S = 0.05, 30
    cast = _f32 if dtype == "f32" else (lambda x: x)
    rng = np.random.default_rng(30)
    u0, p = rng.uniform(-2, 2, (2, 1)), cast(R.weights())
    traj = R.restate("ld", R.problem(dt, S, u0, p, {S: 0}, TM.COSTS["scalar"]), sa)["us"][:S, :, 0]   # u_0 .. u_{S-1}
    starts = cast(traj.T)                                            # [2][S]: one window per member
    dLdu = cast(rng.standard_normal((1, 2, S)))
    tol = 1e-14 if dtype == "f64" else 2000 * 2 * EPS32

    def window(cols):
        eng = _engine(sa, len(cols), np.array([dt]), dt, dt, "explicit", dtype)
        _, du0, dp = _run(eng, starts[:, cols], p, dLdu[:, :, cols])
        eng.close()
        ref = R.restate("ld", R.problem(dt, 1, starts[:, cols], p, {1: 0}, "explicit", dLdu[:, :, cols]), sa)
        return du0, dp, ref

    du0, _, ref = window(list(range(S)))
    err = np.abs(du0 - ref["du0"]).max(axis=0) / np.abs(ref["du0"]).max(axis=0)
    print(f"{sa} {dtype}: one-step windows, largest du0 error {err.max():.1e} at step {int(err.argmax())}")
    assert err.max() <= tol, [(n, float(e)) for n, e in enumerate(err) if e > tol]
    for n in (0, 2, S - 1):
        _, dp, ref = window([n])
        e_p, per = R.dp_err(dp, ref["mu"].sum(1))
        print(f"{sa} {dtype}: window {n} dp {e_p:.1e}")
        assert e_p <= (1e-12 if dtype == "f64" else 2000 * 2 * EPS32), (n, per)


# ------------------------------------------------------------------------------------------------------------------------
# geometry


def _cyclic(N, K, seed):
    """u0 of N members repeating K distinct states; -> (u0[2][N], base[2][K], counts[K])"""
    base = np.random.default_rng(seed).uniform(-2, 2, (2, K))
    idx = np.arange(N) % K
    return base[:, idx], base, np.bincount(idx, minlength=K)


SIZES = {"1": lambda nsm: 1, "31": lambda nsm: 31, "32": lambda nsm: 32, "33": lambda nsm: 33, "4113": lambda nsm: 4096 + 17,
         "64nsm+1": lambda nsm: 64 * nsm + 1}


@pytest.mark.parametrize("size", list(SIZES))
def test_ensemble_sizes(size):
    """GaussAdjoint, dt = 0.25, per-component affine cost, events on; members cycle through 37 distinct states"""
    N = SIZES[size](_nsm())
    K = min(N, 37)
    dt, T = 0.25, TM.T_END
    S = 6
    u0, base, cnt = _cyclic(N, K, 5)
    grid = np.arange(S + 1) * dt
    ev = TM.event_table(S)
    eng = _engine("gauss", N, grid, dt, T, "vector", events=TM.device_events(ev, dt))
    _, du0, dp = _run(eng, u0, R.weights())
    eng.close()
    ref = R.restate("ld", R.problem(dt, S, base, R.weights(), {n: n for n in range(S + 1)}, TM.COSTS["vector"], events=ev), "gauss")
    ref_full = dict(du0=ref["du0"][:, np.arange(N) % K], mu=(ref["mu"] * cnt).sum(1, keepdims=True))
    _report(f"N = {N}", du0, dp, ref_full)


@pytest.mark.parametrize("dtype", ["f64", "f32"])
@pytest.mark.parametrize("sa", ["interpolating", "gauss"])
def test_member_shift_and_block_sums(sa, dtype):
    """(1) a cyclic shift moving every member to another block and another lane leaves saved and du0 bit-identical;
    (2) dp(33 members) = dp(first 32) + dp(last 1) bit for bit: the reduction sums the block partials in block order
    in fp64 from 0, so F64 gives a + b and F32 float(double(a) + double(b)); (3) a repeated reverse() is bitwise the
    same.  dt = 0.25, explicit cost, events on."""
    dt, T, S = 0.25, TM.T_END, 6
    grid = np.arange(S + 1) * dt
    dev_ev = TM.device_events(TM.event_table(S), dt)
    rng = np.random.default_rng(40)
    p = R.weights()
    N, shift = 5 * 32 + 13, 2 * 32 + 5
    pos = (np.arange(N) + shift) % N
    assert ((pos // 32) != (np.arange(N) // 32)).all() and ((pos % 32) != (np.arange(N) % 32)).all()
    u0 = rng.uniform(-2, 2, (2, N))
    dL = rng.standard_normal((S + 1, 2, N))
    order = np.roll(np.arange(N), shift)                    # position q runs member order[q]
    out = []
    for perm in (np.arange(N), order):
        eng = _engine(sa, N, grid, dt, T, "explicit", dtype, events=dev_ev)
        saved, du0, _ = _run(eng, u0[:, perm], p, dL[:, :, perm])
        if perm is order:
            du0b = np.array(eng.reverse(dL[:, :, perm])[0], dtype=np.float64)
            assert np.array_equal(du0, du0b)
        eng.close()
        saved[..., perm] = saved.copy(); du0[:, perm] = du0.copy()
        out.append((saved, du0))
    assert np.array_equal(out[0][0], out[1][0]) and np.array_equal(out[0][1], out[1][1])
    # block sums
    u33, dL33 = u0[:, :33], dL[:, :, :33]
    res = {}
    for key, cols in (("all", slice(0, 33)), ("first", slice(0, 32)), ("last", slice(32, 33))):
        n = len(range(33)[cols])
        eng = _engine(sa, n, grid, dt, T, "explicit", dtype, events=dev_ev)
        _, _, dp = _run(eng, u33[:, cols], p, dL33[:, :, cols])
        if key == "all":
            dp2 = np.array(eng.reverse(dL33[:, :, cols])[1], dtype=np.float64)
            assert np.array_equal(dp, dp2)                   # repeated reverse: same bits
        eng.close()
        res[key] = dp
    if dtype == "f64":
        expect = res["first"] + res["last"]
    else:
        expect = (res["first"] + res["last"]).astype(np.float32).astype(np.float64)
    assert np.array_equal(res["all"], expect), np.abs(res["all"] - expect).max()


@pytest.mark.parametrize("sa", ["interpolating", "gauss"])
def test_c4_at_production_size(sa):
    """BASELINE C4: 4096 members, dt = 0.05, saveat = 0.05 .. 1.5 (30 saves), scalar affine cost, F64; members cycle
    through 61 distinct states: every du0 and all of dp against the restatement"""
    N, K, dt, T, S = 4096, 61, 0.05, 1.5, 30
    saveat = np.linspace(0.05, T, 30)
    u0, base, cnt = _cyclic(N, K, 61)
    p = R.weights()
    eng = _engine(sa, N, saveat, dt, T, "scalar")
    _, du0, dp = _run(eng, u0, p)
    eng.close()
    ref = R.restate("ld", R.problem(dt, S, base, p, {n: n - 1 for n in range(1, S + 1)}, TM.COSTS["scalar"]), sa)
    _report(f"C4 {sa}", du0, dp, dict(du0=ref["du0"][:, np.arange(N) % K], mu=(ref["mu"] * cnt).sum(1, keepdims=True)))
