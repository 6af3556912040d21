"""The bf16 twin of tests/mlp_bf16_twin.py on its own, without a GPU.

* Exact mode against the long-double restatement (mlp_restatement.restate('ld')): pairwise over sensealg x {scalar,
  per-component, explicit} cost x {plain, no_start} x dt in {0.05, 0.25}.  du0 to 1e-15, dp to 1e-13 with the block
  floors of mlp_restatement.dp_err.
* The twin's bf16 rounding against torch's CPU bfloat16 cast, bit for bit: ties, both signs, values next to powers of
  two, subnormals, overflow to infinity, and random bit patterns.
* Bf16 mode against the fp64 restatement at BASELINE C4's bound of 2e-2: a sanity check of the contract.
* The separation guards: every wrong variant lies at least 10x the derived bound away from the twin at the configurations of
  tests/test_gpu_mlp_bf16_reference.py that must catch it (its whole-gradient rows and its Gauss window gradients), on
  both layouts.
"""
import os
import sys

import numpy as np
import pytest

HERE = os.path.dirname(os.path.abspath(__file__))
if HERE not in sys.path:
    sys.path.insert(0, HERE)

import mlp_bf16_twin as T
import mlp_restatement as R
import test_gpu_mlp_bf16_reference as G
import test_mlp_restatement as TM

# (sensealg, cost, mode, dt): a pairwise cover of the four factors
EXACT_CASES = [("interpolating", "scalar", "plain", 0.05), ("interpolating", "vector", "no_start", 0.25),
               ("interpolating", "explicit", "plain", 0.25), ("gauss", "scalar", "no_start", 0.25),
               ("gauss", "vector", "plain", 0.05), ("gauss", "explicit", "no_start", 0.05)]


def _setup(sa, cost, mode, dt, M=5, seed=0, amp=2.0):
    """saves at every grid point of [0, 1.5], t0 included; -> (problem of the restatement, run() arguments)"""
    S = int(round(TM.T_END / dt))
    rng = np.random.default_rng(seed)
    u0 = T.f32(rng.uniform(-amp, amp, (2, M)))
    p = T.f32(R.weights())
    sos = {n: n for n in range(S + 1)}
    dLdu = T.f32(rng.standard_normal((S + 1, 2, M))) if cost == "explicit" else None
    c = TM.COSTS[cost]
    pr = R.problem(dt, S, u0, p, sos, c, dLdu, no_start=mode == "no_start")
    return pr, dict(p=p, u0=u0, h=dt, S=S, sos=sos, cost=c, dLdu=dLdu, sensealg=sa, no_start=mode == "no_start")


@pytest.mark.parametrize("case", EXACT_CASES, ids=lambda c: "-".join(map(str, c)))
def test_exact_mode_matches_the_long_double_restatement(case):
    pr, kw = _setup(*case)
    ref = R.restate("ld", pr, case[0])
    tw = T.run(mode="exact", **kw)
    e_u = np.abs(tw["du0"] - ref["du0"]).max() / np.abs(ref["du0"]).max()
    e_p, per = R.dp_err(tw["dp"], ref["mu"].sum(1))
    e_s = np.abs(tw["us"] - ref["us"]).max() / np.abs(ref["us"]).max()
    print(f"{case}: us {e_s:.1e} du0 {e_u:.1e} dp {e_p:.1e}")
    assert e_s <= 1e-15 and e_u <= 1e-15, (e_s, e_u)
    assert e_p <= 1e-13, per


def test_bf16_rounding_matches_torch_bit_for_bit():
    import torch
    rng = np.random.default_rng(1)
    one = np.float32(1.0).view(np.uint32)
    pats = [np.arange(0, 1 << 16, dtype=np.uint32) << 16 | 0x8000,            # exact ties at every bf16 value: even / odd
            (np.arange(0, 1 << 16, dtype=np.uint32) << 16) | 0x7FFF,           # just below a tie
            (np.arange(0, 1 << 16, dtype=np.uint32) << 16) | 0x8001,           # just above a tie
            rng.integers(0, 1 << 32, 200000, dtype=np.uint64).astype(np.uint32)]
    x = np.concatenate([p.view(np.float32) for p in pats])
    # next to powers of two (both sides), subnormals, the largest finite values, both signs
    pw = np.exp2(np.arange(-149, 128, dtype=np.float64)).astype(np.float32)
    near = np.concatenate([np.nextafter(pw, np.float32(0)), pw, np.nextafter(pw, np.float32(np.inf))])
    sub = (np.arange(1, 1 << 12, dtype=np.uint32) * 2039).view(np.float32)
    big = np.array([np.finfo(np.float32).max, np.float32(3.3961e38), np.float32(3.389e38)], dtype=np.float32)
    x = np.concatenate([x, near, sub, big, np.float32([0.0, 1.0, 0.5])])
    x = np.concatenate([x, -x])
    x = x[np.isfinite(x)]
    assert one == 0x3F800000
    ours = np.asarray(T.bf16(x), dtype=np.float32).view(np.uint32)
    ref = torch.from_numpy(x).to(torch.bfloat16).to(torch.float32).numpy().view(np.uint32)
    bad = np.flatnonzero(ours != ref)
    assert bad.size == 0, [(hex(x.view(np.uint32)[i]), hex(ours[i]), hex(ref[i])) for i in bad[:10]]
    # round toward zero truncates
    assert np.array_equal(np.asarray(T.bf16(x, rz=True), dtype=np.float32).view(np.uint32), x.view(np.uint32) & 0xFFFF0000)


@pytest.mark.parametrize("sa", ["interpolating", "gauss"])
@pytest.mark.parametrize("layout", ["narrow", "wide"])
def test_bf16_mode_within_the_c4_bound(sa, layout):
    """C4's grid (dt = 0.05, S = 30), scalar affine cost: the bf16 twin within 2e-2 of the fp64 restatement"""
    pr, kw = _setup(sa, "scalar", "plain", 0.05, M=8, seed=2)
    ref = R.restate("ld", pr, sa)
    tw = T.run(layout=layout, **kw)
    e_s = np.abs(tw["us"] - ref["us"]).max() / np.abs(ref["us"]).max()
    e_u = np.abs(tw["du0"] - ref["du0"]).max() / np.abs(ref["du0"]).max()
    e_p = {k: np.abs(tw["dp"][sl] - ref["mu"].sum(1)[sl]).max() / np.abs(ref["mu"].sum(1)[sl]).max() for k, sl in R.BLOCKS.items()}
    print(f"{sa} {layout}: us {e_s:.1e} du0 {e_u:.1e} dp " + " ".join(f"{k} {v:.1e}" for k, v in e_p.items()))
    assert e_s < 1e-2 and e_u < 1e-2 and max(e_p.values()) < 2e-2


# ------------------------------------------------------------------------------------------------------------------------
# separation guards, at the configurations of tests/test_gpu_mlp_bf16_reference.py (its inputs, its seeds, an H100's 132
# SMs for the layout), with the twin's own trajectory and np.tanh rounded to fp32 standing in for the kernel's


NSM = 132


def _whole_row(**want):
    return next(c for c in G.WHOLE if all(c["sa cost mode dt size".split().index(k)] == v for k, v in want.items()))


# variant -> the whole-gradient rows of the GPU file that must catch it, one per layout
WHOLE_GUARDS = {
    "cost_component0": [_whole_row(cost="vector", size="33"), _whole_row(cost="vector", size="64nsm+1")],
    "no_start_ignored": [_whole_row(mode="no_start", size="33"), _whole_row(mode="no_start", size="64nsm+1")],
    "rz_all": [_whole_row(sa="gauss", cost="scalar", mode="plain", dt=0.05)],
}
# variant -> the dt of test_gauss_window_gradients that must catch it (both layouts).  k6 read for k7 in the reverse
# dense output is not among them: k6 = f at the c = 1 stage and k7 = f(u_{n+1}) differ by the stage's local error, and
# the y it moves (by b_7(theta) h (k7 - k6)) stays within about a tenth of the derived bound at dt = 0.05 and 0.25.
WINDOW_GUARDS = {"mirrored_gauss_nodes": 0.05, "lam_drops_ka6": 0.05, "rz_all": 0.05, "rz_H1": 0.05, "rz_dZ2": 0.05}


@pytest.mark.parametrize("c", [(v, c) for v, cs in WHOLE_GUARDS.items() for c in cs], ids=lambda vc: f"{vc[0]}-{G._whole_label(vc[1])}")
def test_whole_gradient_separation_guard(c):
    variant, row = c
    w = G.whole_inputs(*row, NSM)
    layout = "narrow" if -(-w["N"] // 32) <= 2 * NSM else "wide"
    us = T.run(w["p"], w["base"], row[3], w["S"], {}, TM.COSTS["scalar"], layout=layout)["us"]
    base, bounds = T.derive(G.whole_runner(row, w, us=us, layout=layout))
    wrong = G.whole_runner(row, w, us=us, layout=layout, variant=variant)(None)
    sep = max(T.ratios({"du0": wrong["du0"], "dp": wrong["dp"]}, base, bounds).values())
    print(f"{variant} at {G._whole_label(row)} ({layout}): {sep:.1f} x the derived bound")
    assert sep >= 10, sep


@pytest.mark.parametrize("layout", ["narrow", "wide"])
@pytest.mark.parametrize("variant", list(WINDOW_GUARDS))
def test_window_separation_guard(variant, layout):
    dt = WINDOW_GUARDS[variant]
    p, u0, dLdu = G.window_inputs(dt)
    starts = T.run(p, u0, dt, G.WINDOW_K, {}, TM.COSTS["scalar"])["us"][:G.WINDOW_K, :, 0].T
    N = G.WINDOW_K if layout == "narrow" else 64 * NSM + 1
    cnt = np.bincount(np.arange(N) % G.WINDOW_K, minlength=G.WINDOW_K)
    base, bounds = T.derive(G.window_runner(p, starts, dt, dLdu, cnt, layout=layout))
    wrong = G.window_runner(p, starts, dt, dLdu, cnt, layout=layout, variant=variant)(None)
    sep = max(T.ratios({"du0": wrong["du0"], "dp": wrong["dp"]}, base, bounds).values())
    print(f"{variant} at Gauss windows dt {dt} ({layout}): {sep:.1f} x the derived bound")
    assert sep >= 10, sep
