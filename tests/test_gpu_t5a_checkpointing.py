"""Checkpointed save intervals on the adaptive Tsit5 path (B200ADJ_FLAG_CHECKPOINT_SAVES): the forward pass keeps one step
state per member and save interval, the reverse kernel re-solves each interval with the forward kernel's own step.  The
gradient must be the full-storage mode's gradient BIT FOR BIT (np.array_equal, no tolerance), for every family, sensealg,
parameter layout, cost and save-time layout; the memory the handle owns must follow the documented formula to the byte."""
import os

import numpy as np
import pytest

pytestmark = pytest.mark.gpu

import scimlsensitivity_jl_b200 as b
from scimlsensitivity_jl_b200 import _lib

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
UNSUPPORTED = -2
P_OF = {"lv": np.array([1.5, 1.0, 3.0, 1.0]), "lorenz": np.array([10.0, 28.0, 8.0 / 3.0]), "vanderpol": np.array([1.0, 1.0])}
U0_OF = {"lv": np.array([1.0, 1.0]), "lorenz": np.array([1.0, 0.0, 0.0]), "vanderpol": np.array([2.0, 0.0])}


def _register(name, **kw):
    """The plug-ins are prebuilt in-tree by __graft_entry__.build(); a stale one is rebuilt here."""
    so = os.path.join(ROOT, "examples", f"libb200fam_{name}.so")
    if os.path.exists(so):
        try:
            return b.register_family(so)
        except b.B200AdjError:
            os.remove(so)
    header, struct = kw.pop("header"), kw.pop("struct")
    return b.register_family(b.build_family_plugin(os.path.join(ROOT, "examples", header), struct, name, out=so, **kw))


@pytest.fixture(scope="module")
def vdp():
    return _register("vanderpol", header="vanderpol_family.cuh", struct="VanDerPol", has_jac=False)


def _inputs(family, N, shared_p, seed=0):
    rng = np.random.default_rng(seed)
    d = len(U0_OF[family])
    u0 = U0_OF[family][:, None] * np.exp(0.1 * rng.standard_normal((d, N))) + (0.05 * rng.standard_normal((d, N)) if family == "lorenz" else 0.0)
    p = P_OF[family] if shared_p else P_OF[family][:, None] * np.exp(0.05 * rng.standard_normal((len(P_OF[family]), N)))
    return u0, np.ascontiguousarray(p)


def _pair(family, N, saveat, T, tol, shared_p, max_steps=(4096, 4096), cost=None):
    """(full, checkpointed) engines with the same configuration"""
    kw = dict(shared_p=shared_p, abstol=tol, reltol=tol, cost=cost if cost is not None else b.AffineCost(1.0, -2.0))
    full = b.DeviceEnsemble(family, "interpolating", "tsit5_adaptive", N, saveat, (0.0, T), 0.0, max_steps=max_steps[0], **kw)
    ck = b.DeviceEnsemble(family, "interpolating", "tsit5_adaptive", N, saveat, (0.0, T), 0.0, max_steps=max_steps[1], checkpoint_saves=True, **kw)
    return full, ck


def _forward_equal(full, ck, u0, p):
    sf, stf = full.forward(u0, p)
    sc, stc = ck.forward(u0, p)
    assert np.array_equal(stf, stc) and (stf == 0).all()
    assert np.array_equal(sf, sc)
    assert np.array_equal(full.step_counts()[0], ck.step_counts()[0])
    return sf


COSTS = ("explicit", "affine", "affine_vec_dgdp", "continuous")


def _reverse_both(engs, sensealg, cost, saveat, d, P, N, no_start=False, seed=1):
    """the same reverse pass on every engine -> [(du0, dp)]"""
    rng = np.random.default_rng(seed)
    dLdu = rng.standard_normal((len(saveat), d, N))
    out = []
    for e in engs:
        e.handle.set_continuous_cost(cost == "continuous", 0.3, -0.2)
        if cost == "explicit":
            e.set_reverse(sensealg, cost=None, no_start=no_start, t=saveat)
            du0, dp = e.reverse(dLdu)
        elif cost == "affine_vec_dgdp":
            e.set_reverse(sensealg, cost=b.AffineCost(np.linspace(0.5, 1.5, d), np.linspace(-1.0, 1.0, d)), no_start=no_start, t=saveat,
                          dgdp=b.ParamAffine(np.linspace(0.1, 0.4, P), np.linspace(1.0, -1.0, P)))
            du0, dp = e.reverse()
        else:
            e.set_reverse(sensealg, cost=b.AffineCost(1.0, -2.0), no_start=no_start, t=saveat)
            du0, dp = e.reverse()
        out.append((du0.copy(), dp.copy()))
    return out


def _assert_bitwise(res):
    (du0f, dpf), (du0c, dpc) = res
    assert np.isfinite(du0f).all() and np.isfinite(dpf).all()
    assert np.array_equal(du0f, du0c), np.abs(du0f - du0c).max()
    assert np.array_equal(dpf, dpc), np.abs(dpf - dpc).max()


@pytest.mark.parametrize("shared_p", [True, False])
@pytest.mark.parametrize("family,tol", [("lv", 1e-5), ("lv", 1e-10), ("lorenz", 1e-7), ("lorenz", 1e-10), ("vanderpol", 1e-6), ("vanderpol", 1e-9)])
def test_bitwise_matrix(family, tol, shared_p, vdp):
    """every sensealg x cost (x no_start) on one forward pass of each mode; tolerances 1e-5..1e-10 reject steps"""
    N, T = 96, (3.0 if family == "lorenz" else 8.0)
    saveat = np.linspace(0.0, T, 13)
    d, P = len(U0_OF[family]), len(P_OF[family])
    u0, p = _inputs(family, N, shared_p)
    full, ck = _pair(family, N, saveat, T, tol, shared_p)
    _forward_equal(full, ck, u0, p)
    for k, sensealg in enumerate(("interpolating", "gauss", "gauss_kronrod")):
        for j, cost in enumerate(COSTS):
            _assert_bitwise(_reverse_both((full, ck), sensealg, cost, saveat, d, P, N, no_start=(j + k) % 2 == 1, seed=10 * k + j))
    full.close(); ck.close()


LAYOUTS = {
    "t0_and_t1": lambda T: np.linspace(0.0, T, 11),
    "inside_only": lambda T: np.linspace(0.0, T, 12)[1:-1],
    "t1_only": lambda T: np.array([T]),                               # one interval
    "dense_200": lambda T: np.linspace(0.3 * T, 0.35 * T, 200),       # many save times inside one step: intervals share straddling steps
    "off_grid_ends": lambda T: np.array([0.0, 0.37 * T, 0.371 * T, T]),
}


@pytest.mark.parametrize("layout", sorted(LAYOUTS))
@pytest.mark.parametrize("sensealg", ["interpolating", "gauss", "gauss_kronrod"])
def test_save_time_layouts(layout, sensealg):
    N, T, tol = 64, 8.0, 1e-8
    saveat = LAYOUTS[layout](T)
    for shared_p in (True, False):
        u0, p = _inputs("lv", N, shared_p, seed=5)
        full, ck = _pair("lv", N, saveat, T, tol, shared_p)
        _forward_equal(full, ck, u0, p)
        for cost in ("explicit", "affine"):
            _assert_bitwise(_reverse_both((full, ck), sensealg, cost, saveat, 2, 4, N))
        full.close(); ck.close()


def test_c1_ensemble_bitwise_and_memory():
    """bench.py's C1 ensemble (65 536 members, tol 1e-8, K = 101): full mode at max_steps = 512 against 64 steps per interval"""
    N, T = 65536, 10.0
    saveat = np.linspace(0.0, T, 101)
    u0 = np.exp(0.2 * np.random.default_rng(3000).standard_normal((2, N)))
    full, ck = _pair("lv", N, saveat, T, 1e-8, True, max_steps=(512, 64), cost=b.AffineCost(0.0, 1.0))
    _forward_equal(full, ck, u0, P_OF["lv"])
    for sensealg in ("interpolating", "gauss"):
        res = []
        for e in (full, ck):
            e.set_reverse(sensealg, cost=b.AffineCost(0.0, 1.0), t=saveat)
            du0, dp = e.reverse()
            res.append((du0.copy(), dp.copy()))
        _assert_bitwise(res)
    bf, bc = full.device_bytes(), ck.device_bytes()
    assert bc * 4 < bf, (bc, bf)
    full.close(); ck.close()


def test_interval_capacity_status_2():
    """per-member p: one member needs more steps in one save interval than max_steps -> status 2 and NaN gradients; every other
    member is bitwise the full mode's"""
    N, T, tol = 64, 10.0, 1e-8
    saveat = np.linspace(0.0, T, 11)
    u0, p = _inputs("lv", N, False, seed=7)
    p[:, 0] *= 60.0                                                   # member 0: sixty times the rates
    full = b.DeviceEnsemble("lv", "interpolating", "tsit5_adaptive", N, saveat, (0.0, T), 0.0, shared_p=False, abstol=tol, reltol=tol,
                            cost=b.AffineCost(1.0, -2.0), max_steps=1 << 15)
    sf, stf = full.forward(u0, p)
    assert (stf == 0).all()
    nf = full.step_counts()[0]
    cap = int(nf[1:].max())                        # one interval never needs more steps than the member's whole solve
    assert nf[0] > 10 * (cap + 2)                  # member 0 cannot fit one of its ten intervals into that
    ck = b.DeviceEnsemble("lv", "interpolating", "tsit5_adaptive", N, saveat, (0.0, T), 0.0, shared_p=False, abstol=tol, reltol=tol,
                          cost=b.AffineCost(1.0, -2.0), max_steps=cap, checkpoint_saves=True)
    sc, stc = ck.forward(u0, p)
    assert stc[0] == 2 and (stc[1:] == 0).all()
    assert np.array_equal(sf[:, :, 1:], sc[:, :, 1:])
    for sensealg in ("interpolating", "gauss", "gauss_kronrod"):
        (du0f, dpf), (du0c, dpc) = _reverse_both((full, ck), sensealg, "affine", saveat, 2, 4, N)
        assert np.isnan(du0c[:, 0]).all() and np.isnan(dpc[:, 0]).all()
        assert np.array_equal(du0f[:, 1:], du0c[:, 1:]) and np.array_equal(dpf[:, 1:], dpc[:, 1:])
    full.close(); ck.close()


def _bytes_formula(N, d, P, K, MS, nsm, nseg=None):
    """b200adj_device_bytes of an adaptive Tsit5 handle with buffers_on_device = 1 and no events (include/b200adj.h)"""
    qgrid = min((N + 3) // 4, 6 * nsm)
    total = N * (MS + 1) * (8 * d + 5) * 8 + 12 * N + 2 * max(K, 1) * 8 + max(qgrid + 1, (N + 31) // 32) * P * 8 + 4
    if nseg is not None:
        total += N * nseg * (2 * d + 4) * 8
    return total


@pytest.mark.parametrize("family,N,MS,layout", [("lv", 1000, 300, "t0_and_t1"), ("lorenz", 4097, 77, "inside_only"),
                                                ("lv", 65536, 64, "t0_and_t1"), ("lorenz", 33, 4096, "dense_200")])
def test_device_bytes_formula(family, N, MS, layout):
    import torch
    nsm = torch.cuda.get_device_properties(0).multi_processor_count
    T = 5.0
    saveat = LAYOUTS[layout](T)
    d, P = len(U0_OF[family]), len(P_OF[family])
    nseg = 1 + int(((saveat > 0.0) & (saveat < T)).sum())
    for ckp in (False, True):
        e = b.DeviceEnsemble(family, "interpolating", "tsit5_adaptive", N, saveat, (0.0, T), 0.0, on_device=True, max_steps=MS,
                             abstol=1e-8, reltol=1e-8, cost=b.AffineCost(1.0, 0.0), checkpoint_saves=ckp)
        assert e.device_bytes() == _bytes_formula(N, d, P, len(saveat), MS, nsm, nseg if ckp else None)
        e.close()
    if (N, MS) == (65536, 64):                     # the C1 shape: 64 steps per interval, against the full mode at 512
        full = _bytes_formula(N, d, P, len(saveat), 512, nsm)
        assert _bytes_formula(N, d, P, len(saveat), 64, nsm, nseg) * 4 < full


# ---- refusals: every path / sensealg / setter the mode does not carry is B200ADJ_ERR_UNSUPPORTED, naming the flag ----

def _ck_engine(family="lv", sensealg="interpolating", stepper="tsit5_adaptive", saveat=None, **kw):
    T = 2.0
    saveat = np.linspace(0.0, T, 5) if saveat is None else saveat
    dt = 0.0 if stepper == "tsit5_adaptive" or stepper == "rosenbrock23" else 0.01
    return b.DeviceEnsemble(family, sensealg, stepper, 8, saveat, (0.0, T), dt, abstol=1e-8, reltol=1e-8, cost=b.AffineCost(1.0, 0.0),
                            checkpoint_saves=True, **kw)


def _run(e):
    d, P = e.d, e.P
    u0 = np.full((d, e.N), 0.5) if e.family != "mlp" else None
    p = np.full(P, 1.0)
    e.forward(u0, p)
    du0, dp = e.reverse()
    assert np.isfinite(du0).all() and np.isfinite(dp).all()


CREATE_ROWS = [
    ("lv", "interpolating", "tsit5_adaptive", {}, 0),
    ("lv", "gauss", "tsit5_adaptive", {}, 0),
    ("lv", "gauss_kronrod", "tsit5_adaptive", {}, 0),
    ("lv", "backsolve", "tsit5_adaptive", {}, UNSUPPORTED),
    ("lv", "quadrature", "tsit5_adaptive", {}, UNSUPPORTED),
    ("lv", "interpolating", "rosenbrock23", {}, UNSUPPORTED),
    ("lv", "interpolating", "tsit5_fixed", {}, UNSUPPORTED),                       # fixed step grid
    ("lv", "interpolating", "tsit5_fixed", {"dense_forward": True}, UNSUPPORTED),  # dense fixed-step framework
    ("sde_lv", "interpolating", "em", {}, UNSUPPORTED),
    ("mlp", "interpolating", "tsit5_fixed", {}, UNSUPPORTED),
]


@pytest.mark.parametrize("family,sensealg,stepper,kw,code", CREATE_ROWS, ids=[f"{r[0]}-{r[1]}-{r[2]}-{len(r[3])}" for r in CREATE_ROWS])
def test_refusals_at_create(family, sensealg, stepper, kw, code):
    if code == 0:
        _run(_ck_engine(family, sensealg, stepper, **kw))
        return
    with pytest.raises(b.B200AdjError) as ei:
        _ck_engine(family, sensealg, stepper, **kw)
    assert ei.value.code == code and "CHECKPOINT_SAVES" in str(ei.value)


def _setter_rows():
    T = 2.0
    same = np.linspace(0.0, T, 5)
    return [
        ("set_reverse backsolve", lambda e: e.set_reverse("backsolve", cost=b.AffineCost(1.0, 0.0), t=same), UNSUPPORTED),
        ("set_reverse quadrature", lambda e: e.set_reverse("quadrature", cost=b.AffineCost(1.0, 0.0), t=same), UNSUPPORTED),
        ("set_reverse other times", lambda e: e.set_reverse("gauss", cost=b.AffineCost(1.0, 0.0), t=np.linspace(0.0, T, 7)), UNSUPPORTED),
        ("set_reverse fewer times", lambda e: e.set_reverse("gauss", cost=b.AffineCost(1.0, 0.0), t=same[1:]), UNSUPPORTED),
        ("set_reverse same times", lambda e: e.set_reverse("gauss_kronrod", cost=b.AffineCost(1.0, 0.0), t=same), 0),
        ("set_reverse K < 0", lambda e: e.handle.set_reverse_options(_lib.SA["gauss"], _lib.COST["affine"], 1.0, 0.0, 0, None), 0),
        ("set_events E > 0", lambda e: e.set_events([0.7], [[1.0, 1.0]], [[0.1, 0.0]]), UNSUPPORTED),
        ("set_events E = 0", lambda e: e.set_events([], None, None), 0),
        ("set_continuous_callback", lambda e: e.handle.set_continuous_callback(0, 0.5, -1), UNSUPPORTED),
        ("set_continuous_callback off", lambda e: e.handle.set_continuous_callback(0, enabled=False), 0),
        ("set_continuous_cost", lambda e: e.handle.set_continuous_cost(True, 0.5, 0.0), 0),
    ]


@pytest.mark.parametrize("row", range(len(_setter_rows())), ids=[r[0] for r in _setter_rows()])
def test_refusals_at_setters(row):
    name, call, code = _setter_rows()[row]
    e = _ck_engine()
    if code == 0:
        call(e)
        _run(e)
    else:
        with pytest.raises(b.B200AdjError) as ei:
            call(e)
        assert ei.value.code == code and "CHECKPOINT_SAVES" in str(ei.value), name
        _run(e)                                    # the refused call left the handle usable
    e.close()


def test_refusal_family_events():
    """VectorContinuousCallback with the family's own conditions: refused on a checkpointed handle"""
    fid = _register("projectile", header="vector_callback_families.cuh", struct="ProjectileWall", has_events=True)[0]
    nc = _lib.family_conditions(fid)
    assert nc > 0
    e = b.DeviceEnsemble("projectile", "interpolating", "tsit5_adaptive", 8, np.linspace(0.0, 1.0, 5), (0.0, 1.0), 0.0, abstol=1e-8,
                         reltol=1e-8, cost=b.AffineCost(1.0, 0.0), checkpoint_saves=True)
    with pytest.raises(b.B200AdjError) as ei:
        e.handle.set_family_events(nc, np.zeros(nc, np.int32), 16)
    assert ei.value.code == UNSUPPORTED and "CHECKPOINT_SAVES" in str(ei.value)
    e.handle.set_family_events(nc, np.zeros(nc, np.int32), 16, enabled=False)      # switching it off is accepted
    e.close()


# ---- the public API: solve + adjoint_sensitivities / the rrule with B200Adjoint(..., checkpoint_saves=True) ----

@pytest.mark.parametrize("inner", ["gauss", "interpolating"])
def test_public_api_bitwise(inner):
    N, T = 128, 10.0
    saveat = np.linspace(0.0, T, 21)
    u0, _ = _inputs("lv", N, True, seed=11)
    p = P_OF["lv"]
    alg = b.Tsit5(adaptive=True)
    mk = (lambda: b.GaussAdjoint()) if inner == "gauss" else (lambda: b.InterpolatingAdjoint())
    res = []
    for ckp in (False, True):
        b.clear_handle_cache()
        prob = b.EnsembleProblem(b.ODEProblem("lv", u0[:, 0], (0.0, T), p), u0s=u0)
        sa = b.B200Adjoint(mk(), checkpoint_saves=ckp)
        sol = b.solve(prob, alg, b.EnsembleB200(device=0), saveat=saveat, sensealg=sa, abstol=1e-9, reltol=1e-9)
        du0, dp = b.adjoint_sensitivities(sol, alg, t=saveat, dgdu_discrete=b.AffineCost(1.0, -2.0), sensealg=sa, abstol=1e-9, reltol=1e-9)
        out, back = b._concrete_solve_adjoint(prob, alg, sa, u0, p, None, saveat=saveat, abstol=1e-9, reltol=1e-9)
        grads = back(np.ones_like(np.asarray(out.u)))
        res.append((np.asarray(sol.u).copy(), np.asarray(du0).copy(), np.asarray(dp).copy(), np.asarray(grads[3]).copy(), np.asarray(grads[4]).copy()))
    for a, c in zip(*res):
        assert np.array_equal(a, c)
    b.clear_handle_cache()
