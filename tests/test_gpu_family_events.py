"""VectorContinuousCallback on the device: the conditions and affect compiled into a family plug-in
(examples/vector_callback_families.cuh, B200ADJ_FAMILY_HAS_EVENTS), found by the adaptive Tsit5 forward kernel and
differentiated by the reverse kernels with the implicit event-time correction of src/callback_tracking.jl:232-480.

The four testsets of the reference's test/Callbacks2/vector_continuous_callbacks.jl are restated on their own systems.  The
reference's testset 1 keeps the default save_positions = (true, true), so its loss also sums the states saved at each event;
here the loss is the saveat-only one (save_positions = (false, false) is the mode carried on the device), and the relation
the reference checks -- adjoint = differentiation through the solve -- is checked against closed forms: the flights are
polynomials of degree <= 2 with a nilpotent adjoint system, which Tsit5 integrates exactly.
"""
import os
import sys
import tempfile

import numpy as np
import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
import scimlsensitivity_jl_b200 as b
from scimlsensitivity_jl_b200 import _lib
from scimlsensitivity_jl_b200.problems import FAMILY_CONDITIONS
from oracle import oracle as O

HEADER = os.path.join(ROOT, "examples", "vector_callback_families.cuh")
# struct -> (family name, NC)
EVENT_FAMILIES = {"ProjectileWall": ("projectile", 2), "ClockReset": ("clock_reset", 2), "TiedWalls": ("tied_walls", 2),
                  "CornerWalls": ("corner_walls", 2), "BallEvents": ("ball_events", 1), "RelaxEvents": ("relax_events", 1),
                  "VanDerPolRing": ("vdp_ring", 1)}
SENSEALGS = ["interpolating", "gauss", "gauss_kronrod", "backsolve"]
TOL = dict(abstol=1e-10, reltol=1e-10)


def _register(struct):
    name = EVENT_FAMILIES[struct][0]
    so = b.build_family_plugin(HEADER, struct, name, out=os.path.join(ROOT, "examples", f"libb200fam_{name}.so"), has_events=True)
    b.register_family(so)
    return name


@pytest.fixture(scope="module")
def families():
    return {s: _register(s) for s in EVENT_FAMILIES}


def _rel(a, ref):
    a, ref = np.asarray(a), np.asarray(ref)
    return float(np.max(np.abs(a - ref)) / (np.max(np.abs(ref)) + 1e-300))


# ---------------------------------------------------------------- CPU: build and registration (no marker)

def test_every_example_struct_builds_with_events_and_reports_its_conditions(families):
    for struct, (name, nc) in EVENT_FAMILIES.items():
        assert FAMILY_CONDITIONS[name] == nc
        assert _lib.family_conditions(_lib.FAM[name]) == nc
    for fam, fid in _lib.FAM.items():
        if fid < 100:
            assert _lib.family_conditions(fid) == 0, fam          # every built-in family has none


def test_plugin_without_the_events_macro_still_builds():
    with tempfile.TemporaryDirectory() as tmp:
        so = b.build_family_plugin(HEADER, "BallEvents", "ball_events_plain", out=os.path.join(tmp, "libb200fam_ball_events_plain.so"))
        fid, d, P = b.register_family(so)
        assert (d, P) == (2, 2) and _lib.family_conditions(fid) == 0
        assert FAMILY_CONDITIONS["ball_events_plain"] == 0


# ---------------------------------------------------------------- closed forms

def _projectile(u0, p, ts, T=10.0):
    """ProjectileWall: states at ts and the event list [(t, condition, direction)] for one member (complex-step safe)."""
    x0, v0, y0, w0 = u0
    g, e = p
    floors, tl, xs, vs = [], 0.0, x0, v0
    while True:
        s = (vs + np.sqrt(vs * vs + 2 * g * xs)) / g
        if (tl + s).real > T:
            break
        floors.append((tl, xs, vs, tl + s))
        tl, xs, vs = tl + s, 0.0 * x0, -e * (vs - g * s)
    tw = (10.0 - y0) / w0
    out = []
    for t in ts:
        ta, xa, va = 0.0, x0, v0
        for (a_, xa_, va_, tb_) in floors:
            if t > tb_.real:
                ta, xa, va = tb_, 0.0 * x0, -e * (va_ - g * (tb_ - a_))
        s = t - ta
        x, v = xa + va * s - 0.5 * g * s * s, va - g * s
        y, w = (y0 + w0 * t, w0) if t < tw.real else (10.0 - e * w0 * (t - tw), -e * w0)
        out.append([x, v, y, w])
    evs = sorted([(f[3], 0, -1) for f in floors] + ([(tw, 1, +1)] if tw.real < T else []), key=lambda z: np.real(z[0]))
    return np.array(out), evs


def _clock(u0, p, ts):
    """ClockReset: u .= [0.5, 1, 0, 0] at every k pi / 2."""
    g = p[0]
    out = []
    for t in ts:
        k = int(np.floor(t / (np.pi / 2)))
        if k == 0:
            x0, v0, y0, w0, ta = u0[0], u0[1], u0[2], u0[3], 0.0
        else:
            x0, v0, y0, w0, ta = 0.5 + 0 * g, 1.0 + 0 * g, 0.0 * g, 0.0 * g, k * np.pi / 2
        s = t - ta
        out.append([x0 + v0 * s - 0.5 * g * s * s, v0 - g * s, y0 + w0 * s, w0 + 0 * s])
    return np.array(out)


def _complex_step_grad(loss, x):
    h = 1e-30
    gr = np.zeros(len(x))
    for j in range(len(x)):
        xc = np.array(x, dtype=complex)
        xc[j] += 1j * h
        gr[j] = loss(xc).imag / h
    return gr


def _mse(states):
    return np.sum((states - 1.0) ** 2) / 2


def _projectile_inputs(N, seed=11):
    rng = np.random.default_rng(seed)
    r = lambda: rng.uniform(-1, 1, N)
    u0 = np.stack([50.0 + 0.2 * r(), 0.05 * r(), 0.005 * (1 + r()), 2.01 + 0.003 * r()])
    p = np.stack([9.8 + 0.02 * r(), 0.9 + 0.003 * r()])
    u0[:, 0] = [50.0, 0.0, 0.0, 2.01]; p[:, 0] = [9.8, 0.9]          # the reference's member
    return u0, p


# ---------------------------------------------------------------- GPU

def _engine(fam, sa, N, ts, tspan, cb, shared_p=False, cost=None, every=False, **kw):
    eng = b.DeviceEnsemble(fam, sa, "tsit5_adaptive", N, ts, tspan, 0.0, cost=cost, shared_p=shared_p, ckpt_every_step=every, **{**TOL, **kw})
    eng.set_continuous_callback(cb)
    return eng


def _ball_inputs(N, shared_p, seed=3):
    rng = np.random.default_rng(seed)
    u0 = np.stack([50.0 + 5.0 * rng.standard_normal(N), 0.5 * rng.standard_normal(N)])
    p = np.array([9.8, 0.8]) if shared_p else np.stack([9.8 + 0.3 * rng.standard_normal(N), 0.8 + 0.03 * rng.standard_normal(N)])
    return u0, p


@pytest.mark.gpu
@pytest.mark.parametrize("shared_p", [True, False])
@pytest.mark.parametrize("sa", SENSEALGS)
def test_ball_events_family_path_equals_the_named_path(families, sa, shared_p):
    """BallEvents carries the built-in ball's named callback as family conditions.  Both run the same event search and
    saltation with operands equal value for value, so the forward outputs are bitwise equal.  The gradients agree to a few
    ulps (1.2e-15 of the largest du0 with per-member p on an H100), not bitwise: the two kernels are compiled separately."""
    N = 48
    u0, p = _ball_inputs(N, shared_p)
    t = np.linspace(0.5, 15.0, 30)
    every = sa == "backsolve"
    named = _engine("ball", sa, N, t, (0.0, 15.0), b.ContinuousCallback(idx=0, direction=-1, p_comp=1, p_param=1, p_sign=-1.0, max_events=32),
                    shared_p=shared_p, cost=b.AffineCost(1.0, 0.0), every=every)
    fam = _engine(families["BallEvents"], sa, N, t, (0.0, 15.0), b.VectorContinuousCallback(direction=-1, max_events=32),
                  shared_p=shared_p, cost=b.AffineCost(1.0, 0.0), every=every)
    s1, st1 = named.forward(u0, p); g1 = named.reverse(); c1, t1 = named.event_times()
    s2, st2 = fam.forward(u0, p); g2 = fam.reverse(); c2, t2 = fam.event_times()
    assert (np.asarray(st1) == 0).all() and np.array_equal(np.asarray(st1), np.asarray(st2))
    assert np.array_equal(c1, c2) and c1.min() >= 3
    mask = np.arange(t1.shape[0])[:, None] < c1[None, :]
    assert np.array_equal(t1[mask], t2[mask]) and np.array_equal(np.asarray(s1), np.asarray(s2))
    print(f"{sa} shared_p={shared_p}: du0 rel {_rel(g2[0], g1[0]):.1e}, dp rel {_rel(g2[1], g1[1]):.1e}")
    assert _rel(g2[0], g1[0]) < 2e-15 and _rel(g2[1], g1[1]) < 2e-15
    flags = fam.event_flags()
    assert flags.shape == (32, 1, N) and (flags[:, 0][mask] == -1).all() and (flags[:, 0][~mask] == 0).all()
    cfg = O.make_cfg("ball", sa, "tsit5_adaptive", N, t, 0.0, 15.0, cost=("affine", 1.0, 0.0), shared_p=shared_p, ckpt_every_step=every,
                     crossing=dict(idx=0, level=0.0, direction=-1, pcomp=1, pparam=1, psign=-1.0), **TOL)
    ref = O.gradient(cfg, t, u0, p)
    for g in (g1, g2):
        assert _rel(g[0], ref["du0"]) < 1e-7 and _rel(g[1], ref["dp"]) < 1e-7


GND = np.array([0.9999546000702386, 0.00018159971904994378])      # test/Callbacks2/continuous_callbacks.jl:343


@pytest.mark.gpu
@pytest.mark.parametrize("shared_p", [True, False])
@pytest.mark.parametrize("sa", SENSEALGS)
def test_relax_events_reproduce_gND(families, sa, shared_p):
    """condition u - 3/4 p[1], affect u += p[2] as family conditions: u(10) = p1 + (p2 - p1/4) 4 e^-10 from u0 = 0, so every
    member's gradient is the printed gND."""
    N = 40
    rng = np.random.default_rng(5)
    p = np.array([100.0, 50.0]) if shared_p else np.stack([100.0 + 20.0 * rng.random(N), 50.0 + 10.0 * rng.random(N)])
    eng = _engine(families["RelaxEvents"], sa, N, np.array([10.0]), (0.0, 10.0), b.VectorContinuousCallback(direction=0),
                  shared_p=shared_p, every=True, abstol=1e-14, reltol=1e-14)
    saved, status = eng.forward(np.zeros((1, N)), p)
    du0, dp = eng.reverse(np.ones((1, 1, N)))
    counts, times = eng.event_times()
    assert (np.asarray(status) == 0).all() and (counts == 1).all()
    assert np.max(np.abs(times[0] - np.log(4.0))) < 1e-12
    rtol = 1e-6 if sa == "gauss_kronrod" else 1e-10
    dp = np.asarray(dp)
    if shared_p:
        assert np.allclose(dp.ravel() / N, GND, rtol=rtol, atol=0), dp.ravel() / N - GND
    else:
        assert np.allclose(dp, GND[:, None], rtol=rtol, atol=0), np.abs(dp - GND[:, None]).max(axis=1)


@pytest.mark.gpu
@pytest.mark.parametrize("sa", SENSEALGS)
def test_projectile_wall_against_the_closed_form(families, sa):
    """"callback with linear affect": floor (t ~ 3.19), wall (10 / 2.01 ~ 4.98), floor (~ 8.94) for every member."""
    N = 64
    u0, p = _projectile_inputs(N)
    ts = np.arange(0.0, 10.0 + 1e-12, 0.5)
    eng = _engine(families["ProjectileWall"], sa, N, ts, (0.0, 10.0), b.VectorContinuousCallback(), cost=b.AffineCost(1.0, -1.0),
                  every=sa == "backsolve")
    saved, status = eng.forward(u0, p)
    du0, dp = eng.reverse()
    counts, times = eng.event_times()
    flags = eng.event_flags()
    assert (np.asarray(status) == 0).all() and (counts == 3).all()
    for i in range(N):
        ref, evs = _projectile(u0[:, i], p[:, i], ts)
        assert [(c, d) for _, c, d in evs] == [(0, -1), (1, +1), (0, -1)]
        assert np.min(np.abs(np.array([e[0] for e in evs])[:, None] - ts[None, :])) > 0.01       # no event on a save time
        assert np.allclose(times[:3, i], [e[0] for e in evs], rtol=1e-12, atol=0)
        assert [tuple(flags[k, :, i]) for k in range(3)] == [(-1, 0), (0, 1), (-1, 0)]
        assert _rel(np.asarray(saved)[:, :, i], ref) < 1e-10
        x = np.concatenate([u0[:, i], p[:, i]])
        gr = _complex_step_grad(lambda z: _mse(_projectile(z[:4], z[4:], ts)[0]), x)
        assert _rel(np.asarray(du0)[:, i], gr[:4]) < 1e-8, (i, np.asarray(du0)[:, i], gr[:4])
        assert _rel(np.asarray(dp)[:, i], gr[4:]) < 1e-8, (i, np.asarray(dp)[:, i], gr[4:])


@pytest.mark.gpu
@pytest.mark.parametrize("sa", SENSEALGS)
def test_clock_reset_against_the_closed_form(families, sa):
    """"condition that depends on time only": sin t, cos t; events at k pi / 2, each a full reset."""
    N = 16
    u0, p = _projectile_inputs(N, seed=4)
    ts = np.arange(0.0, 10.0 + 1e-12, 0.5)
    eng = _engine(families["ClockReset"], sa, N, ts, (0.0, 10.0), b.VectorContinuousCallback(), cost=b.AffineCost(1.0, -1.0),
                  every=sa == "backsolve")
    saved, status = eng.forward(u0, p)
    du0, dp = eng.reverse()
    counts, times = eng.event_times()
    assert (np.asarray(status) == 0).all() and (counts == 6).all()
    assert np.allclose(times[:6], (np.pi / 2 * np.arange(1, 7))[:, None], rtol=1e-12, atol=0)
    flags = eng.event_flags()
    assert [tuple(flags[k, :, 0]) for k in range(6)] == [(0, -1), (-1, 0), (0, 1), (1, 0), (0, -1), (-1, 0)]
    for i in range(N):
        assert _rel(np.asarray(saved)[:, :, i], _clock(u0[:, i], p[:, i], ts)) < 1e-10
        gr = _complex_step_grad(lambda z: _mse(_clock(z[:4], z[4:], ts)), np.concatenate([u0[:, i], p[:, i]]))
        assert np.allclose(np.asarray(du0)[:, i], gr[:4], rtol=1e-8, atol=1e-8 * np.abs(gr).max())
        assert _rel(np.asarray(dp)[:, i], gr[4:]) < 1e-8


def _walls(u0, T):
    """TiedWalls from [x, y, vx, vy] with vx < 0: x = 0 at tau, then vy <- vx, vx <- -vx; -> state at T."""
    x0, y0, vx, vy = u0
    tau = -x0 / vx
    return np.array([-vx * (T - tau), y0 + vy * tau + vx * (T - tau), -vx, vx])


@pytest.mark.gpu
@pytest.mark.parametrize("sa", SENSEALGS)
def test_tied_walls_fire_together_and_match_the_closed_form(families, sa):
    """"structural simultaneous fire": u[1] and 2 u[1] land on the same bits at every event; loss at t1 only (:148)."""
    N = 16
    rng = np.random.default_rng(7)
    u0 = np.array([3.0, 1.0, -1.0, 0.0])[:, None] + 0.05 * rng.uniform(-1, 1, (4, N))
    u0[:, 0] = [3.0, 1.0, -1.0, 0.0]
    T = 5.0
    eng = _engine(families["TiedWalls"], sa, N, [T], (0.0, T), b.VectorContinuousCallback(), shared_p=True, every=sa == "backsolve")
    saved, status = eng.forward(u0, np.array([0.0]))
    uT = np.asarray(saved)[0]
    dL = np.zeros((1, 4, N)); dL[0, :2] = 2 * (uT[:2] - 0.5)
    du0, dp = eng.reverse(dL)
    counts, _ = eng.event_times()
    flags = eng.event_flags()
    assert (np.asarray(status) == 0).all() and (counts == 1).all()
    assert (flags[0] == -1).all()                                   # both conditions, downwards
    for i in range(N):
        assert _rel(uT[:, i], _walls(u0[:, i], T)) < 1e-12
        gr = _complex_step_grad(lambda z: np.sum((_walls(z, T)[:2] - 0.5) ** 2), u0[:, i])
        assert np.allclose(np.asarray(du0)[:, i], gr, rtol=1e-8, atol=1e-8 * np.abs(gr).max()), (i, np.asarray(du0)[:, i], gr)


@pytest.mark.gpu
@pytest.mark.parametrize("sa", SENSEALGS)
def test_corner_walls_trap_fires_both_and_gives_finite_gradients(families, sa):
    """"corner trap" at the reference's u0: both walls flagged at t = 1, du0 finite, two runs bitwise equal."""
    N = 4
    u0 = np.tile(np.array([[1.0], [1.0], [-1.0], [-1.0]]), (1, N))
    res = []
    for _ in range(2):
        eng = _engine(families["CornerWalls"], sa, N, [3.0], (0.0, 3.0), b.VectorContinuousCallback(), shared_p=True, every=sa == "backsolve")
        saved, status = eng.forward(u0, np.array([0.0]))
        uT = np.asarray(saved)[0].copy()
        dL = np.zeros((1, 4, N)); dL[0, :2] = 2 * (uT[:2] - 0.5)
        du0, dp = eng.reverse(dL)
        counts, times = eng.event_times()
        flags = eng.event_flags()
        assert (np.asarray(status) == 0).all() and (counts == 1).all() and np.allclose(times[0], 1.0, rtol=1e-12)
        assert (flags[0] == -1).all()
        assert np.isfinite(np.asarray(du0)).all()
        res.append((uT, np.asarray(du0).copy(), np.asarray(dp).copy()))
    assert all(np.array_equal(x, y) for x, y in zip(*res))


@pytest.mark.gpu
@pytest.mark.parametrize("sa", SENSEALGS)
def test_vanderpol_ring_against_finite_differences(families, sa):
    """Non-polynomial flow, p-dependent condition |u|^2 - p3^2 (direction +1), affect u <- u / 2, per-member p: adjoint against
    central differences of the device's own forward pass."""
    N = 16
    rng = np.random.default_rng(9)
    u0 = np.stack([0.5 + 0.05 * rng.uniform(-1, 1, N), 0.05 * rng.uniform(-1, 1, N)])
    p = np.stack([1.0 + 0.05 * rng.uniform(-1, 1, N), 1.0 + 0.05 * rng.uniform(-1, 1, N), 1.5 + 0.05 * rng.uniform(-1, 1, N)])
    ts = np.arange(0.5, 8.0 + 1e-12, 0.5)
    kw = dict(abstol=1e-12, reltol=1e-12)
    cb = b.VectorContinuousCallback(direction=+1)
    eng = _engine(families["VanDerPolRing"], sa, N, ts, (0.0, 8.0), cb, cost=b.AffineCost(1.0, 0.0), every=sa == "backsolve", **kw)
    saved, status = eng.forward(u0, p)
    du0, dp = eng.reverse()
    counts, _ = eng.event_times()
    assert (np.asarray(status) == 0).all() and counts.min() >= 1
    fd_eng = _engine(families["VanDerPolRing"], "gauss", N, ts, (0.0, 8.0), cb, cost=b.AffineCost(1.0, 0.0), **kw)

    def loss(u, q):
        s, st = fd_eng.forward(u, q)
        assert (np.asarray(st) == 0).all()
        return 0.5 * np.sum(np.asarray(s) ** 2, axis=(0, 1))
    x = np.concatenate([u0, p])
    fd = np.zeros_like(x)
    for j in range(5):
        h = 1e-6 * np.maximum(1.0, np.abs(x[j]))
        xp, xm = x.copy(), x.copy()
        xp[j] += h; xm[j] -= h
        fd[j] = (loss(xp[:2], xp[2:]) - loss(xm[:2], xm[2:])) / (2 * h)
    adj = np.concatenate([np.asarray(du0), np.asarray(dp)])
    for j in range(5):
        assert np.max(np.abs(adj[j] - fd[j])) <= 2e-5 * np.max(np.abs(fd[j])) + 1e-9, (j, adj[j], fd[j])


def _code(fn):
    try:
        fn()
    except _lib.B200AdjError as e:
        return e.code
    return 0


@pytest.mark.gpu
def test_status_codes_of_the_family_event_entry_points(families):
    proj = families["ProjectileWall"]
    ts = np.array([1.0, 2.0])
    mk = lambda fam, sa="gauss", st="tsit5_adaptive", dt=0.0: b.DeviceEnsemble(fam, sa, st, 4, ts, (0.0, 2.0), dt)
    UNS, INV, STATE = -2, -1, -5
    dirs = np.zeros(2, np.int32)
    # the family carries no conditions: every built-in family
    for fam in ("ball", "lv"):
        assert _code(lambda: mk(fam).handle.set_family_events(1, np.zeros(1, np.int32), 8)) == UNS
    assert _code(lambda: mk("sde_lv", "backsolve", "em", 0.01).handle.set_family_events(1, np.zeros(1, np.int32), 8)) == UNS
    # not adaptive Tsit5
    assert _code(lambda: mk(proj, st="tsit5_fixed", dt=0.01).handle.set_family_events(2, dirs, 8)) == UNS
    # preset-time events, both orders
    e = mk(proj)
    e.set_events([0.5], [[1, 1, 1, 1]], [[0, 0, 0, 0]])
    assert _code(lambda: e.handle.set_family_events(2, dirs, 8)) == UNS
    e = mk(proj)
    e.handle.set_family_events(2, dirs, 8)
    assert _code(lambda: e.handle.set_events([0.5], [[1, 1, 1, 1]], [[0, 0, 0, 0]])) == UNS
    # QuadratureAdjoint: on the entry point and in set_reverse_options
    assert _code(lambda: mk(proj, "quadrature").handle.set_family_events(2, dirs, 8)) == UNS
    assert _code(lambda: e.set_reverse("quadrature", cost=b.AffineCost(1.0, 0.0))) == UNS
    # invalid arguments
    e = mk(proj)
    assert _code(lambda: e.handle.set_family_events(1, np.zeros(1, np.int32), 8)) == INV
    assert _code(lambda: e.handle.set_family_events(2, np.array([0, 2], np.int32), 8)) == INV
    assert _code(lambda: e.handle.set_family_events(2, dirs, 0)) == INV
    # state
    e.handle.set_family_events(2, dirs, 8)
    assert _code(lambda: e.handle.event_flags(4, 8)) == STATE
    assert _code(lambda: e.handle.set_continuous_callback_params(lparam=0, lcoef=1.0)) == STATE
    assert _code(lambda: _lib.family_conditions(99)) == INV
    # enabled = 0 removes it; set_continuous_callback switches to the named mode
    e.handle.set_family_events(2, dirs, 8, enabled=False)
    assert _code(lambda: e.handle.event_times(4, 8)) == STATE


@pytest.mark.gpu
def test_public_api_solve_and_pullback_match_the_closed_form(families):
    N = 32
    u0, p = _projectile_inputs(N, seed=21)
    prob = b.ODEProblem(families["ProjectileWall"], u0[:, 0], (0.0, 10.0), p[:, 0], callback=b.VectorContinuousCallback())
    eprob = b.EnsembleProblem(prob, u0s=u0)
    ts = np.arange(0.0, 10.0 + 1e-12, 0.5)
    sol = b.solve(eprob, b.Tsit5(adaptive=True), b.EnsembleB200(), saveat=0.5, u0=u0, p=p, **TOL)
    out, pullback = b._concrete_solve_adjoint(eprob, b.Tsit5(adaptive=True), b.B200Adjoint(b.GaussAdjoint()), u0, p, None, saveat=0.5, **TOL)
    assert np.array_equal(np.asarray(sol.u), np.asarray(out.u))
    tang = pullback(np.asarray(out.u) - 1.0)
    du0, dp = tang[3], tang[4]
    for i in range(N):
        ref, _ = _projectile(u0[:, i], p[:, i], ts)
        assert _rel(np.asarray(out.u)[:, :, i], ref) < 1e-10
        gr = _complex_step_grad(lambda z: _mse(_projectile(z[:4], z[4:], ts)[0]), np.concatenate([u0[:, i], p[:, i]]))
        assert _rel(np.asarray(du0)[:, i], gr[:4]) < 1e-8 and _rel(np.asarray(dp)[:, i], gr[4:]) < 1e-8
