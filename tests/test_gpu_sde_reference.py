"""Whole gradients of the SDE kernels (csrc/sde_em.cuh) against the restatement of tests/sde_restatement.py, with the
increments the device exported (get_noise) on both sides.

* The configuration matrix of tests/sde_restatement.py (both families x EM / EulerHeun x Backsolve with each checkpoint
  mode and Interpolating with and without no_start x scalar affine, vector affine plus dgdp, explicit cost x shared and
  per-member p x regenerated, stored and caller-supplied noise x saveat the full grid, a subset without t0, a subset
  without T and a single point; every pair of levels and every sde_backsolve_kernel instantiation that disp_sde.cu can
  launch, each COST_EXPLICIT one included): du0 and dp per member and component at 1e-12 relative, the component floored
  at 1e-6 of the member's largest, in 40 digits for 3 members and in long double for all 96 (the shared-p dp as the sum
  over the members; long double agrees with 40 digits to 1e-15 on the 3).  Where a component cancels (a dp of a noise
  parameter summed from terms of both signs, an explicit cotangent), no float64 evaluation of the algorithm meets
  1e-12 of it: the bound is then 4x the float64 restatement's own distance from long double (it was needed in 4 of
  the 32 configurations, at most 6.2e-12), and a dp with a dgdp part is measured against the larger of its two summands.
* The tolerance separates the kernel from near misses: the device lies >= 100 bounds from the restatement with the
  1/2-factor Ito correction, with the reverse increment +dW_{n-1} or -dW_n, with the Interpolating EulerHeun corrector at
  y(t_n), and with the Backsolve checkpoint reset after the loss jump.
* Launch geometry: block_threads 32, 96, 160, 224, 512 x N = 1, 33, block + 1, 3 block - 5, shared p (the cross-block
  store_dp ticket reduction), against long double; a second reverse pass of the same forward pass is bitwise identical.
* The host state machine of api.cu: forward(dW=X) -> reverse -> forward() -> reverse follows the Philox stream the
  second time; a get_noise call between forward and reverse leaves the gradients bit-identical; set_reverse on one forward
  pass switches Backsolve -> Interpolating -> Backsolve(checkpointing=False) -> explicit cost with retargeted t and more
  save times than at creation (the staging buffer of dL/du reallocated).
* C5 at full size (N = 131 072, EM dt = 0.01, BacksolveAdjoint, Philox noise regenerated): 64 sampled members through
  the long-double restatement, du0 per member, and dp per member from the same run with per-member p.

Observed on an H100 80GB HBM3 (700 W power limit), largest error as a share of its bound: whole gradients 0.86 (in 40
digits at most 3.2e-14, 0.032), launch geometry 0.36, set_reverse 0.27, C5 members 0.083.  The near misses lie 4e10
(reset after the jump) to 5e13 bounds away.  The module took 17 s of host time there.
"""
import os
import sys

import numpy as np
import pytest

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(HERE)
for d in (ROOT, HERE):
    if d not in sys.path:
        sys.path.insert(0, d)

import sde_restatement as R

pytestmark = pytest.mark.gpu
TOL = 1e-12
N_MATRIX = 96
OBS = {}


def _seen(kind, share):
    OBS[kind] = max(OBS.get(kind, 0.0), float(share))
    print(f"OBSERVED {kind}: {OBS[kind]:.3g} of the bound")


def _engine(c, N, seed=0, traj_offset=0, block_threads=0, saveat=None):
    import scimlsensitivity_jl_b200 as b
    u0, p, cost, dgdp, dLdu = R.problem(c, N, seed=seed)
    sensealg, ckpt, no_start = R.SENSEALGS[c["sa"]]
    saveat = R.SAVEATS[c["saveat"]] if saveat is None else saveat
    acost = None if cost[0] == "explicit" else b.AffineCost(cost[1], cost[2])
    kw = dict(no_start=no_start, checkpointing=ckpt != "never", ckpt_every_step=ckpt == "every")
    eng = b.DeviceEnsemble(c["family"], sensealg, c["stepper"], N, saveat, (0.0, R.T_END), R.H, shared_p=c["p"] == "shared",
                           cost=acost, stored_noise=c["noise"] == "stored", seed=1000 + seed, traj_offset=traj_offset,
                           block_threads=block_threads, **kw)
    if dgdp is not None:
        eng.set_reverse(sensealg, cost=acost, dgdp=b.ParamAffine(dgdp[0], dgdp[1]), **kw)
    return eng, (u0, p, cost, dgdp, dLdu)


def _run(c, N, seed=0, **kw):
    """-> (du0, dp, dW, inputs) of one device run"""
    eng, inp = _engine(c, N, seed=seed, **kw)
    u0, p, cost, dgdp, dLdu = inp
    dW_in = np.sqrt(R.H) * np.random.default_rng(seed + 1).standard_normal((R.S_STEPS, 2, N)) if c["noise"] == "dW" else None
    _, status = eng.forward(u0, p, dW=dW_in)
    assert (np.asarray(status) == 0).all()
    dW = np.array(eng.noise())
    if dW_in is not None:
        assert np.array_equal(dW, dW_in)
    du0, dp = [np.array(x) for x in eng.reverse(dLdu)]
    du0b, dpb = eng.reverse(dLdu)
    assert np.array_equal(du0, du0b) and np.array_equal(dp, dpb)
    eng.close()
    return du0, dp, dW, inp


def _restated(kind, c, inp, dW, idx=None, saveat=None, variant=None, **over):
    u0, p, cost, dgdp, dLdu = inp
    sensealg, ckpt, no_start = R.SENSEALGS[c["sa"]]
    sel = (lambda a: a) if idx is None else (lambda a: a[..., idx])
    pp = p if np.ndim(p) == 1 else sel(p)
    args = dict(cost=cost, dLdu=None if dLdu is None else sel(dLdu), dgdp=dgdp, ckpt=ckpt, no_start=no_start, variant=variant)
    args.update(over)
    return R.gradient(kind, c["family"], c["stepper"], sensealg, sel(u0), pp, sel(dW), R.H,
                      R.SAVEATS[c["saveat"]] if saveat is None else saveat, **args)[:2]


def _dgdp_part(c, inp, saveat=None):
    """the parameter part njump (c p + e) of dp per member (None without dgdp): the jumps applied, all K save times but
    the first under Interpolating with no_start"""
    u0, p, cost, dgdp, dLdu = inp
    if dgdp is None:
        return None
    K = len(R.SAVEATS[c["saveat"]] if saveat is None else saveat) - (1 if c["sa"] == "interp_no_start" else 0)
    pm = np.asarray(p, dtype=np.float64)
    pm = np.repeat(pm[:, None], u0.shape[1], 1) if pm.ndim == 1 else pm
    return K * (np.asarray(dgdp[0])[:, None] * pm + np.asarray(dgdp[1])[:, None])


def _errors(c, du0, dp, ref_du0, ref_dp, idx=None, f64_shared=False, part=None):
    """largest floored relative error of du0 and dp (dp summed over the members under shared p; f64_shared: dp is a
    per-member restatement to be summed too; part: _dgdp_part)"""
    if f64_shared and c["p"] == "shared":
        dp = dp.sum(1)
    sel = (lambda a: a) if idx is None else (lambda a: a[..., idx])
    e = R.rel_err(sel(du0), ref_du0).max()
    if c["p"] == "shared":
        if idx is None:
            e = max(e, R.rel_err(dp, ref_dp.sum(1), None if part is None else part.sum(1)).max())
    else:
        e = max(e, R.rel_err(sel(dp), ref_dp, None if part is None else sel(part)).max())
    return e


def _bound(c, inp, dW, ld, **over):
    """1e-12, or 4x the float64 restatement's own distance from the long-double one where that is larger: the rounding
    of the algorithm itself in float64, which a component that cancels (dp of a noise parameter, a sum of terms of
    both signs) can lift above 1e-12 of the component"""
    f64 = _restated("f64", c, inp, dW, **over)
    return max(TOL, 4 * _errors(c, f64[0], f64[1], ld[0], ld[1], f64_shared=True, part=_dgdp_part(c, inp, over.get("saveat"))))


@pytest.mark.parametrize("c", R.config_matrix(), ids=R.label)
def test_device_matches_the_restatement(c):
    N = N_MATRIX
    du0, dp, dW, inp = _run(c, N, seed=3, traj_offset=2 ** 32 - N // 2)
    idx = np.array([0, N // 2, N - 1])
    mp_ = _restated("mp", c, inp, dW, idx)
    part = _dgdp_part(c, inp)
    e_mp = _errors(c, du0, dp, mp_[0], mp_[1], idx, part=part)
    ld = _restated("ld", c, inp, dW)
    assert R.rel_err(ld[0][:, idx], mp_[0]).max() < 1e-15          # long double stands in for 40 digits
    tol = _bound(c, inp, dW, ld)
    e_ld = _errors(c, du0, dp, ld[0], ld[1], part=part)
    print(f"{R.label(c)}: 40 digits {e_mp:.2e}, long double {e_ld:.2e}, bound {tol:.2e}")
    _seen("whole gradients", max(e_mp, e_ld) / tol)
    assert e_mp < tol and e_ld < tol


NEAR_MISSES = [("half_ito", dict(family="sde_lv", stepper="em", sa="bs_save", cost="scalar", p="member", noise="regen", saveat="full")),
               ("plus_dw", dict(family="sde_lv", stepper="euler_heun", sa="bs_save", cost="scalar", p="member", noise="regen", saveat="full")),
               ("dw_of_step_n", dict(family="sde_linear", stepper="em", sa="interp", cost="scalar", p="member", noise="regen", saveat="full")),
               ("eh_corrector_at_yn", dict(family="sde_lv", stepper="euler_heun", sa="interp", cost="scalar", p="member", noise="regen", saveat="full")),
               ("reset_after_jump", dict(family="sde_lv", stepper="em", sa="bs_save", cost="scalar", p="member", noise="regen", saveat="full"))]


@pytest.mark.parametrize("variant,c", NEAR_MISSES, ids=[v for v, _ in NEAR_MISSES])
def test_tolerance_rejects_near_miss_algorithms(variant, c):
    du0, dp, dW, inp = _run(c, 64, seed=4)
    ok = _restated("ld", c, inp, dW)
    tol = _bound(c, inp, dW, ok)
    assert _errors(c, du0, dp, ok[0], ok[1]) < tol
    bad = _restated("ld", c, inp, dW, variant=variant)
    sep = _errors(c, du0, dp, bad[0], bad[1]) / tol
    print(f"{variant}: the device lies {sep:.3g} bounds from it")
    assert sep >= 100


GEOMETRY = [(b_, n) for b_ in (32, 96, 160, 224, 512) for n in (1, 33, b_ + 1, 3 * b_ - 5)]
GEO_CONFIGS = [dict(family="sde_lv", stepper="em", sa="bs_save", cost="scalar", p="shared", noise="regen", saveat="full"),
               dict(family="sde_linear", stepper="euler_heun", sa="interp", cost="explicit", p="shared", noise="regen", saveat="no_T"),
               dict(family="sde_lv", stepper="euler_heun", sa="bs_every", cost="vector_dgdp", p="shared", noise="stored", saveat="no_t0"),
               dict(family="sde_linear", stepper="em", sa="bs_never", cost="scalar", p="shared", noise="regen", saveat="single")]


@pytest.mark.parametrize("block,N", GEOMETRY, ids=[f"block{b_}-N{n}" for b_, n in GEOMETRY])
def test_launch_geometry(block, N):
    c = GEO_CONFIGS[GEOMETRY.index((block, N)) % len(GEO_CONFIGS)]
    du0, dp, dW, inp = _run(c, N, seed=6, block_threads=block)
    ld = _restated("ld", c, inp, dW)
    tol = _bound(c, inp, dW, ld)
    e = _errors(c, du0, dp, ld[0], ld[1], part=_dgdp_part(c, inp))
    _seen("launch geometry", e / tol)
    assert e < tol


def test_forward_with_dw_then_philox():
    """forward(dW=X) -> reverse -> forward() -> reverse: the second gradient follows the Philox stream, not X"""
    c = dict(family="sde_lv", stepper="em", sa="bs_save", cost="scalar", p="shared", noise="dW", saveat="full")
    N = 64
    eng, inp = _engine(c, N, seed=8)
    X = np.sqrt(R.H) * np.random.default_rng(9).standard_normal((R.S_STEPS, 2, N))
    eng.forward(inp[0], inp[1], dW=X)
    g1 = [np.array(x) for x in eng.reverse()]
    eng.forward(inp[0], inp[1])
    W = np.array(eng.noise())
    g2 = [np.array(x) for x in eng.reverse()]
    eng.close()
    DW, _ = R.increments(1008, 0, N, R.S_STEPS, 2, R.H, "ld")
    assert np.abs(W - DW.astype(np.float64)).max() < 1e-14 and not np.array_equal(W, X)
    r1, r2 = _restated("ld", c, inp, X), _restated("ld", c, inp, W)
    t1, t2 = _bound(c, inp, X, r1), _bound(c, inp, W, r2)
    assert _errors(c, *g1, *r1) < t1 and _errors(c, *g2, *r2) < t2
    assert _errors(c, *g2, *r1) > 100 * t1


@pytest.mark.parametrize("noise", ["regen", "stored"])
def test_get_noise_between_forward_and_reverse_changes_nothing(noise):
    c = dict(family="sde_linear", stepper="euler_heun", sa="bs_save", cost="scalar", p="member", noise=noise, saveat="no_T")
    eng, inp = _engine(c, 40, seed=10)
    eng.forward(inp[0], inp[1])
    g1 = [np.array(x) for x in eng.reverse()]
    eng.forward(inp[0], inp[1])
    eng.noise()
    g2 = [np.array(x) for x in eng.reverse()]
    eng.close()
    assert all(np.array_equal(a, b_) for a, b_ in zip(g1, g2))


def test_set_reverse_switches_on_one_forward_pass():
    """explicit cost at K = 5 -> Interpolating (affine) -> Backsolve(checkpointing=False) -> explicit cost with t
    retargeted to K' = 9 > 5 save times"""
    import scimlsensitivity_jl_b200 as b
    c = dict(family="sde_lv", stepper="euler_heun", sa="bs_save", cost="explicit", p="member", noise="regen", saveat="no_T")
    N = 50
    eng, inp = _engine(c, N, seed=12)
    u0, p, _, _, dLdu = inp
    eng.forward(u0, p)
    W = np.array(eng.noise())
    steps = []
    steps.append((c, None, eng.reverse(dLdu), {}))
    ac = b.AffineCost(1.0, -0.25)
    eng.set_reverse("interpolating", cost=ac)
    ci = dict(c, sa="interp", cost="scalar")
    steps.append((ci, None, eng.reverse(), dict(cost=("affine", 1.0, -0.25), dLdu=None)))
    eng.set_reverse("backsolve", cost=ac, checkpointing=False)
    cn = dict(c, sa="bs_never", cost="scalar")
    steps.append((cn, None, eng.reverse(), dict(cost=("affine", 1.0, -0.25), dLdu=None)))
    t9 = R.GRID[[0, 4, 9, 15, 20, 26, 31, 37, 40]]
    eng.set_reverse("backsolve", cost=None, t=t9)
    d9 = np.random.default_rng(13).standard_normal((9, 2, N))
    steps.append((c, t9, eng.reverse(d9), dict(dLdu=d9)))
    eng.close()
    for cc, t, (du0, dp), over in steps:
        du0, dp = np.array(du0), np.array(dp)
        ld = _restated("ld", cc, inp, W, saveat=t, **over)
        tol = _bound(cc, inp, W, ld, saveat=t, **over)
        e = _errors(cc, du0, dp, ld[0], ld[1])
        print(f"set_reverse {cc['sa']} {cc['cost']} K={len(R.SAVEATS[cc['saveat']] if t is None else t)}: {e:.2e} (bound {tol:.2e})")
        _seen("set_reverse", e / tol)
        assert e < tol


def test_c5_sampled_members_at_full_size():
    import scimlsensitivity_jl_b200 as b
    N, T, dt = 131072, 1.0, 0.01
    t = np.linspace(0.0, T, 101)
    u0, p = np.ones((2, N)), np.array([1.5, 1.0, 3.0, 1.0, 0.1, 0.1])
    idx = np.sort(np.random.default_rng(14).choice(N, 64, replace=False))
    out = {}
    for shared in (True, False):
        eng = b.DeviceEnsemble("sde_lv", "backsolve", "em", N, t, (0.0, T), dt, shared_p=shared, cost=b.AffineCost(0.0, 1.0), seed=20260923)
        _, status = eng.forward(u0, p if shared else np.repeat(p[:, None], N, 1))
        assert (np.asarray(status) == 0).all()
        du0, dp = [np.array(x) for x in eng.reverse()]
        out[shared] = (du0, dp, np.array(eng.noise())[:, :, idx])
        eng.close()
    assert np.array_equal(out[True][2], out[False][2]) and np.array_equal(out[True][0], out[False][0])
    args = ("sde_lv", "em", "backsolve", u0[:, idx], p, out[True][2], dt, t)
    du0r, dpr, _ = R.gradient("ld", *args, cost=("affine", 0.0, 1.0))
    du0f, dpf, _ = R.gradient("f64", *args, cost=("affine", 0.0, 1.0))
    tol = max(TOL, 4 * max(R.rel_err(du0f, du0r).max(), R.rel_err(dpf, dpr).max()))
    e = max(R.rel_err(out[True][0][:, idx], du0r).max(), R.rel_err(out[False][1][:, idx], dpr).max())
    print(f"C5 sampled members: {e:.2e}, bound {tol:.2e}")
    _seen("C5 members", e / tol)
    assert e < tol
