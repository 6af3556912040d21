"""Device VectorContinuousCallback against independent references: the families of tests/csrc/event_reference_families.cuh
(built here into plug-ins) each pin terms of the event-time correction of the adaptive Tsit5 reverse kernel
(t5a_reverse_kernel, FE branch) that the example families leave untested.

  MovingWall       dg/dt = -p2, dg/dp on p1 and p2, an affect that depends on p2 and p3: numpy closed form, complex-step gradient
  Gates8           8 conditions with their own directions, staggered / tied / one-ulp-apart gates: closed form, complex step
  GatedOscillator  non-polynomial flow, condition in (u, p, t), ring condition, state- and p-dependent non-diagonal affect:
                   a 40-digit mpmath reference (exact flow expm(A t) u, bracketed roots, central differences at h = 1e-15)

Neither reference uses an ODE solver or any of the device's or the oracle's logic.  Gradients are compared per member and
per component: |dev - ref| <= rtol |ref| + 1e-10 max|ref of that member|.
"""
import math
import os
import sys
from concurrent.futures import ThreadPoolExecutor

import mpmath as mp
import numpy as np
import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
import scimlsensitivity_jl_b200 as b
from scimlsensitivity_jl_b200 import _lib
from scimlsensitivity_jl_b200.problems import FAMILY_CONDITIONS

HEADER = os.path.join(ROOT, "tests", "csrc", "event_reference_families.cuh")
EXAMPLES = os.path.join(ROOT, "examples", "vector_callback_families.cuh")
# struct -> (header, family name, NC)
PLUGINS = {"MovingWall": (HEADER, "ref_moving_wall", 1), "Gates8": (HEADER, "ref_gates8", 8),
           "GatedOscillator": (HEADER, "ref_gated_osc", 2), "CornerWalls": (EXAMPLES, "ref_corner_walls", 2)}
# (sensealg, ckpt_every_step)
SENSEALGS = [("interpolating", False), ("gauss", False), ("gauss_kronrod", False), ("backsolve", True), ("backsolve", False)]
SA_IDS = ["interpolating", "gauss", "gauss_kronrod", "backsolve_every_step", "backsolve_saveat"]
N = 257                     # ragged past one 256-thread block


@pytest.fixture(scope="module")
def plugins(tmp_path_factory):
    out = tmp_path_factory.mktemp("event_plugins")
    with ThreadPoolExecutor(max_workers=len(PLUGINS)) as pool:
        sos = dict(zip(PLUGINS, pool.map(lambda s: b.build_family_plugin(PLUGINS[s][0], s, PLUGINS[s][1], has_events=True,
                                                                          out=str(out / f"libb200fam_{PLUGINS[s][1]}.so")), PLUGINS)))
    for so in sos.values():
        b.register_family(so)
    return {s: PLUGINS[s][1] for s in PLUGINS}


# ---------------------------------------------------------------- closed forms (numpy, complex-step safe)

def moving_wall(u0, p, ts, T):
    """MovingWall: states at ts and events [(t, {0: -1})].  From (ta, xa, va) with gap c0 = x - wall >= 0 the impact is
    the positive root of c0 + (va - p2) s - p0 s^2 / 2; then x = wall, v <- p2 - p3 (v - p2)."""
    g, w0, s, e = p
    ta, xa, va, c0 = 0.0 * u0[0], u0[0], u0[1], u0[0] - w0
    segs, events = [(ta, xa, va)], []
    while True:
        vr = va - s
        tau = (vr + np.sqrt(vr * vr + 2 * g * c0)) / g
        if (ta + tau).real > T:
            break
        ta = ta + tau
        vb = va - g * tau
        xa, va, c0 = w0 + s * ta, s - e * (vb - s), 0.0 * c0
        segs.append((ta, xa, va)); events.append((ta, {0: -1}))
    out = []
    for t in ts:
        ta, xa, va = [sg for sg in segs if sg[0].real < t][-1]
        d = t - ta
        out.append([xa + va * d - 0.5 * g * d * d, va - g * d])
    return np.array(out), events


GATE_LEVELS = [1.0, 0.0, 0.3, 0.3000001, 0.55, 0.55, 0.8, float(np.nextafter(0.8, 1.0))]
GATE_DIRS = [+1, -1, 0, +1, -1, 0, 0, 0]


def gates8(u0, p, ts, T):
    """Gates8: piecewise linear motion; the next event is the nearest level ahead whose direction admits the crossing, all
    conditions at that level fire together (the one-ulp pair are two events here, ulp / v apart)."""
    x, v, t = u0[0], u0[1], 0.0 * u0[0]
    segs, events = [(t, x, v)], []
    while True:
        up = v.real > 0
        cand = [(c, (GATE_LEVELS[c] - x) / v) for c in range(8)
                if GATE_DIRS[c] in ((0, 1) if up else (0, -1)) and ((GATE_LEVELS[c] > x.real) if up else (GATE_LEVELS[c] < x.real))]
        if not cand:
            break
        dt = min(cand, key=lambda z: z[1].real)[1]
        if (t + dt).real > T:
            break
        lev = GATE_LEVELS[min(cand, key=lambda z: z[1].real)[0]]
        fired = {c: (1 if up else -1) for c, _ in cand if GATE_LEVELS[c] == lev}
        t = t + dt
        x = lev + 0.0 * x
        for c in fired:
            v = v * (-p[c] if c < 2 else p[c])
        segs.append((t, x, v)); events.append((t, fired))
    out = []
    for ti in ts:
        ta, xa, va = [sg for sg in segs if sg[0].real < ti][-1]
        out.append([xa + va * (ti - ta), va])
    return np.array(out), events


def complex_step_grad(loss, x):
    h = 1e-30
    gr = np.zeros(len(x))
    for j in range(len(x)):
        xc = np.array(x, dtype=complex)
        xc[j] += 1j * h
        gr[j] = loss(xc).imag / h
    return gr


def affine_loss(states, b_):
    """the loss whose dL/du is AffineCost(1, b_): sum (u + b_)^2 / 2 over the save times"""
    return np.sum((states + b_) ** 2) / 2


# ---------------------------------------------------------------- 40-digit reference (mpmath)

DPS = 40


class MpFamily:
    """exact flow, conditions, directions and affect of a family in mpmath"""

    def __init__(self, nc, dirs, flow, cond, affect, delta):
        self.nc, self.dirs, self.flow, self.cond, self.affect, self.delta = nc, dirs, flow, cond, affect, delta


def _osc_flow(u, p, t, dt):
    ed, c, s = mp.exp(-p[0] * dt), mp.cos(p[1] * dt), mp.sin(p[1] * dt)          # expm([[-a, w], [-w, -a]] dt)
    return [ed * (c * u[0] + s * u[1]), ed * (-s * u[0] + c * u[1])]


def _osc_affect(ev, u, p):
    u = list(u)
    if ev.get(0):
        u[1] = u[1] - u[0] * u[1] / 2 + p[4] * u[0]
    if ev.get(1):
        u = [mp.mpf("1.25") * u[0], mp.mpf("1.25") * u[1]]
    return u


def _gates_affect(ev, u, p):
    k = mp.mpf(1)
    for c in ev:
        k *= -p[c] if c < 2 else p[c]
    return [u[0], k * u[1]]


MP_FAMILIES = {
    "GatedOscillator": MpFamily(2, [0, -1], _osc_flow,
                                lambda u, p, t: [u[0] - p[2] * mp.cos(t), u[0] ** 2 + u[1] ** 2 - p[3] ** 2], _osc_affect, 0.01),
    "MovingWall": MpFamily(1, [-1], lambda u, p, t, dt: [u[0] + u[1] * dt - p[0] * dt * dt / 2, u[1] - p[0] * dt],
                           lambda u, p, t: [u[0] - p[1] - p[2] * t], lambda ev, u, p: [u[0], p[2] - p[3] * (u[1] - p[2])], 0.01),
    "Gates8": MpFamily(8, GATE_DIRS, lambda u, p, t, dt: [u[0] + u[1] * dt, u[1]],
                       lambda u, p, t: [u[0] - mp.mpf(lv) for lv in GATE_LEVELS], _gates_affect, 0.01),
}


def mp_solve(fam, u0, p, ts, T):
    """Events and states at ts on the exact flow: the first sample interval (width fam.delta) in which a condition changes
    sign in its direction brackets its root (findroot, 40 digits); conditions whose roots agree to 1e-30 fire together.
    Right after an event a condition that fired there takes its side 1e-25 later."""
    with mp.workdps(DPS):
        u, p, t, T = [mp.mpf(x) for x in u0], [mp.mpf(x) for x in p], mp.mpf(0), mp.mpf(T)
        segs, events, just = [(t, u)], [], set()
        at = lambda tt, c, t_, u_: fam.cond(fam.flow(u_, p, t_, tt - t_), p, tt)[c]
        while True:
            gprev = fam.cond(u, p, t)
            for c in just:
                gprev[c] = at(t + mp.mpf("1e-25"), c, t, u)
            tprev, k, hit = t, 1, None
            while hit is None:
                tk = min(t + k * fam.delta, T)
                gk = fam.cond(fam.flow(u, p, t, tk - t), p, tk)
                cross = [c for c in range(fam.nc) if (fam.dirs[c] <= 0 and gprev[c] > 0 and gk[c] <= 0) or
                         (fam.dirs[c] >= 0 and gprev[c] < 0 and gk[c] >= 0)]
                if cross:
                    hit = (tprev, tk, cross, gprev)
                elif tk >= T:
                    break
                tprev, gprev, k = tk, gk, k + 1
            if hit is None:
                break
            lo, hi, cross, gp = hit
            roots = {c: mp.findroot(lambda s, c=c: at(s, c, t, u), (lo, hi), solver="anderson") for c in cross}
            tstar = min(roots.values())
            fired = {c: (1 if gp[c] < 0 else -1) for c in cross if roots[c] - tstar <= mp.mpf("1e-30")}
            um = fam.flow(u, p, t, tstar - t)
            u, t, just = fam.affect(fired, um, p), tstar, set(fired)
            segs.append((t, u)); events.append((t, fired))
        states = []
        for ti in ts:
            ti = mp.mpf(ti)
            ta, ua = [sg for sg in segs if sg[0] < ti][-1]
            states.append(fam.flow(ua, p, ta, ti - ta))
        return states, events


def mp_grad(fam, u0, p, ts, T, b_):
    """dL/d(u0, p) of L = sum (u(ts) + b_)^2 / 2 by central differences at h = 1e-15 on the 40-digit solution"""
    x = [mp.mpf(v) for v in list(u0) + list(p)]
    d = len(u0)
    with mp.workdps(DPS):
        h = mp.mpf("1e-15")

        def loss(z):
            st, _ = mp_solve(fam, z[:d], z[d:], ts, T)
            return mp.fsum((y + b_) ** 2 for s in st for y in s) / 2
        gr = []
        for j in range(len(x)):
            xp, xm = list(x), list(x)
            xp[j] += h; xm[j] -= h
            gr.append(float((loss(xp) - loss(xm)) / (2 * h)))
    return np.array(gr)


# ---------------------------------------------------------------- inputs

T_WALL, TS_WALL = 3.0, np.linspace(0.13, 3.0, 12)
T_GATES, TS_GATES = 3.0, np.linspace(0.11, 3.0, 10)
T_OSC, TS_OSC = 4.0, np.linspace(0.17, 4.0, 9)
OSC_MEMBERS = [0, 1, 2, 3, 31, 32, 100, 200, 254, 255, 256]        # the members the 40-digit reference covers


def wall_inputs(n=N, seed=31):
    rng = np.random.default_rng(seed)
    gap = rng.uniform(1.5, 6.0, n)
    p = np.stack([9.8 + 0.5 * rng.uniform(-1, 1, n), rng.uniform(-0.5, 0.5, n), rng.choice([-1, 1], n) * rng.uniform(0.2, 0.6, n),
                  rng.uniform(0.7, 0.8, n)])
    u0 = np.stack([p[1] + gap, rng.uniform(-3.0, 3.0, n)])
    u0[1, ::37] = 14.0                          # thrown up high: no impact before T
    return u0, p


def gate_inputs(n=N, seed=41):
    rng = np.random.default_rng(seed)
    u0 = np.stack([rng.uniform(0.02, 0.98, n), rng.choice([-1, 1], n) * rng.uniform(0.3, 1.5, n)])
    u0[:, ::29] = np.array([[0.42], [0.02]])   # slow, between two gates: no event
    p = np.concatenate([rng.uniform(0.9, 1.0, (2, n)), rng.uniform(0.95, 1.05, (6, n))])
    return u0, p


def osc_inputs(n=N, seed=51):
    rng = np.random.default_rng(seed)
    u0 = np.stack([1.0 + 0.3 * rng.uniform(-1, 1, n), 0.3 * rng.uniform(-1, 1, n)])
    p = np.stack([rng.uniform(0.15, 0.3, n), rng.uniform(2.0, 3.0, n), rng.uniform(0.2, 0.4, n), rng.uniform(0.5, 0.7, n),
                  rng.uniform(0.1, 0.3, n)])
    return u0, p


def merge_ulp_pair(events, rtol=1e-12):
    """events [(t, {c: dir})]: the one-ulp gates 6 and 7 may fire together or one after the other; either way is one
    event here"""
    out = []
    for t, ev in events:
        if out and set(ev) <= {6, 7} and set(out[-1][1]) <= {6, 7} and not set(ev) & set(out[-1][1]) \
                and abs(t - out[-1][0]) <= rtol * abs(t):
            out[-1] = (out[-1][0], {**out[-1][1], **ev})
        else:
            out.append((t, dict(ev)))
    return out


def device_events(counts, times, flags, i):
    return [(float(times[k, i]), {c: int(flags[k, c, i]) for c in range(flags.shape[1]) if flags[k, c, i]}) for k in range(counts[i])]


# ---------------------------------------------------------------- CPU: the references agree with each other (no marker)

def test_reference_families_build_into_plugins(plugins):
    for struct, (_, name, nc) in PLUGINS.items():
        assert FAMILY_CONDITIONS[name] == nc
        assert _lib.family_conditions(_lib.FAM[name]) == nc


def _real_events(events):
    return [(float(np.real(t)), ev) for t, ev in events]


@pytest.mark.parametrize("fam", ["MovingWall", "Gates8"])
def test_closed_forms_agree_with_the_40_digit_reference(fam):
    closed, inputs, ts, T = {"MovingWall": (moving_wall, wall_inputs, TS_WALL, T_WALL), "Gates8": (gates8, gate_inputs, TS_GATES, T_GATES)}[fam]
    u0, p = inputs()
    for i in (0, 1, 2, 29, 37, 256):
        st, ev = closed(u0[:, i], p[:, i], ts, T)
        mst, mev = mp_solve(MP_FAMILIES[fam], u0[:, i], p[:, i], ts, T)
        ev, mev = merge_ulp_pair(_real_events(ev)), merge_ulp_pair([(float(t), e) for t, e in mev])
        assert [e for _, e in ev] == [e for _, e in mev], i
        assert np.allclose([t for t, _ in ev], [t for t, _ in mev], rtol=1e-14, atol=0), i
        assert np.allclose(st, np.array(mst, dtype=float), rtol=1e-13, atol=1e-14), i


@pytest.mark.parametrize("fam", ["MovingWall", "Gates8"])
def test_complex_step_gradients_agree_with_40_digit_central_differences(fam):
    closed, inputs, ts, T = {"MovingWall": (moving_wall, wall_inputs, TS_WALL, T_WALL), "Gates8": (gates8, gate_inputs, TS_GATES, T_GATES)}[fam]
    u0, p = inputs()
    for i in (1, 2):
        x = np.concatenate([u0[:, i], p[:, i]])
        cs = complex_step_grad(lambda z: affine_loss(closed(z[:2], z[2:], ts, T)[0], -1.0), x)
        cd = mp_grad(MP_FAMILIES[fam], u0[:, i], p[:, i], ts, T, -1)
        assert np.allclose(cs, cd, rtol=1e-11, atol=1e-12 * np.abs(cd).max()), (i, cs, cd)


def test_inputs_keep_events_apart_from_save_times_and_the_end():
    """the chosen members have ragged event counts, zero-event members, and no event within 1e-6 of a save time or of T
    (far above the 1e-12 the event times are held to, so the order of an event and a save time is never in doubt)"""
    for closed, inputs, ts, T in ((moving_wall, wall_inputs, TS_WALL, T_WALL), (gates8, gate_inputs, TS_GATES, T_GATES)):
        u0, p = inputs()
        counts = []
        for i in range(N):
            _, ev = closed(u0[:, i], p[:, i], ts, T)
            tev = np.array([float(np.real(t)) for t, _ in ev])
            counts.append(len(merge_ulp_pair(_real_events(ev))))
            if len(tev):
                assert np.abs(tev[:, None] - np.append(ts, T)[None, :]).min() > 1e-6, (closed.__name__, i)
        counts = np.array(counts)
        assert counts.min() == 0 and counts.max() >= 3 and len(set(counts[:32])) > 1


# ---------------------------------------------------------------- GPU

DIRECTIONS = {"ref_moving_wall": -1, "ref_gates8": GATE_DIRS, "ref_gated_osc": [0, -1], "ref_corner_walls": 0}


def _engine(fam, sa, every, n, ts, T, shared_p=False, cost=None, max_events=64, tol=1e-10):
    eng = b.DeviceEnsemble(fam, sa, "tsit5_adaptive", n, ts, (0.0, T), 0.0, cost=cost, shared_p=shared_p, ckpt_every_step=every,
                           abstol=tol, reltol=tol)
    eng.set_continuous_callback(b.VectorContinuousCallback(direction=DIRECTIONS[fam], max_events=max_events))
    return eng


def _run(eng, u0, p):
    saved, status = eng.forward(u0, p)
    du0, dp = eng.reverse()
    counts, times = eng.event_times()
    flags = eng.event_flags()
    return np.asarray(saved).copy(), np.asarray(status).copy(), np.asarray(du0).copy(), np.asarray(dp).copy(), counts, times, flags


def _check_member_grads(dev, ref, rtol, what):
    """dev, ref: [n_members][components]; every component within rtol |ref| + 1e-10 max|ref of the member|.  Prints the
    largest relative error over the components above 1e-6 max|ref of the member|."""
    worst, bad = 0.0, []
    for i, (d, r) in enumerate(zip(dev, ref)):
        atol = 1e-10 * np.abs(r).max()
        err = np.abs(d - r)
        if not np.all(err <= rtol * np.abs(r) + atol):
            bad.append((i, d, r))
        big = np.abs(r) > 1e-6 * np.abs(r).max()
        worst = max(worst, float(np.max(err[big] / np.abs(r[big]))))
    print(f"{what}: worst relative error {worst:.2e}")
    assert not bad, f"{what}: {len(bad)} members off, first {bad[0]}"
    return worst


def _closed_form_refs(closed, u0, p, ts, T, b_):
    refs = []
    for i in range(u0.shape[1]):
        st, ev = closed(u0[:, i], p[:, i], ts, T)
        gr = complex_step_grad(lambda z: affine_loss(closed(z[:2], z[2:], ts, T)[0], b_), np.concatenate([u0[:, i], p[:, i]]))
        refs.append((np.real(st), merge_ulp_pair(_real_events(ev)), gr))
    return refs


@pytest.fixture(scope="module")
def wall_refs():
    u0, p = wall_inputs()
    return u0, p, _closed_form_refs(moving_wall, u0, p, TS_WALL, T_WALL, -1.0)


@pytest.fixture(scope="module")
def gate_refs():
    u0, p = gate_inputs()
    return u0, p, _closed_form_refs(gates8, u0, p, TS_GATES, T_GATES, -1.0)


@pytest.fixture(scope="module")
def osc_refs():
    u0, p = osc_inputs()
    refs = {}
    for i in OSC_MEMBERS:
        st, ev = mp_solve(MP_FAMILIES["GatedOscillator"], u0[:, i], p[:, i], TS_OSC, T_OSC)
        refs[i] = (np.array(st, dtype=float), [(float(t), e) for t, e in ev], mp_grad(MP_FAMILIES["GatedOscillator"], u0[:, i], p[:, i], TS_OSC, T_OSC, 0))
    return u0, p, refs


def _grad_rtol(sa, base):
    return 1e-6 if sa == "gauss_kronrod" else base


def _check_against(run, refs, members, ev_rtol, st_tol, g_rtol, what, merge=False):
    saved, status, du0, dp, counts, times, flags = run
    assert (status == 0).all()
    for i in members:
        st, ev, _ = refs[i]
        dev = device_events(counts, times, flags, i)
        assert all(t1 < t2 for (t1, _), (t2, _) in zip(dev, dev[1:])), (what, i, "event times not increasing")
        if merge:
            dev = merge_ulp_pair(dev)
        assert [e for _, e in dev] == [e for _, e in ev], (what, i, dev, ev)
        assert np.allclose([t for t, _ in dev], [t for t, _ in ev], rtol=ev_rtol, atol=0), (what, i)
        assert np.allclose(saved[:, :, i], st, rtol=st_tol, atol=st_tol * np.abs(st).max()), (what, i)
    dev = [np.concatenate([du0[:, i], dp[:, i]]) for i in members]
    return _check_member_grads(dev, [refs[i][2] for i in members], g_rtol, what)


@pytest.mark.gpu
@pytest.mark.parametrize("sa,every", SENSEALGS, ids=SA_IDS)
def test_moving_wall_against_the_closed_form(plugins, wall_refs, sa, every):
    """dg/dt = -p2, dg/dp = [0, -1, -t, 0], v+ = p2 - p3 (v- - p2); 257 members, per-member p, 0 to 5 impacts each.
    Observed on an H100 80GB HBM3 (400 W limit): largest relative gradient error 1.2e-9 (Backsolve every step 4.9e-9)."""
    u0, p, refs = wall_refs
    eng = _engine(plugins["MovingWall"], sa, every, N, TS_WALL, T_WALL, cost=b.AffineCost(1.0, -1.0))
    _check_against(_run(eng, u0, p), refs, range(N), 1e-12, 1e-10, _grad_rtol(sa, 1e-8), f"MovingWall {sa}")


@pytest.mark.gpu
@pytest.mark.parametrize("sa,every", SENSEALGS, ids=SA_IDS)
def test_gates8_against_the_closed_form(plugins, gate_refs, sa, every):
    """8 conditions: every event list, its (condition, direction) flags and dp[c] ~ how often gate c fired.  The one-ulp gates
    may fire together or one after the other: their events are merged on both sides before the comparison, and the count
    of times each gate fired is compared as well.  Observed on an H100 80GB HBM3 (400 W limit): largest relative gradient
    error 1.6e-12 (Backsolve every step 4.5e-12)."""
    u0, p, refs = gate_refs
    eng = _engine(plugins["Gates8"], sa, every, N, TS_GATES, T_GATES, cost=b.AffineCost(1.0, -1.0))
    run = _run(eng, u0, p)
    _, _, _, _, counts, times, flags = run
    for i in range(N):
        fired = np.abs(flags[:counts[i], :, i]).sum(axis=0)
        ref = np.zeros(8, int)
        for _, ev in refs[i][1]:
            for c in ev:
                ref[c] += 1
        assert np.array_equal(fired, ref), (i, fired, ref)
    _check_against(run, refs, range(N), 1e-12, 1e-10, _grad_rtol(sa, 1e-8), f"Gates8 {sa}", merge=True)


@pytest.mark.gpu
@pytest.mark.parametrize("sa,every", SENSEALGS, ids=SA_IDS)
def test_gated_oscillator_against_the_40_digit_reference(plugins, osc_refs, sa, every):
    """non-polynomial flow at device tolerance 1e-12 against the 40-digit reference on the members of OSC_MEMBERS; the
    other members must finish with status 0.  Observed on an H100 80GB HBM3 (400 W limit): largest relative gradient error
    3.0e-9 (every sensealg)."""
    u0, p, refs = osc_refs
    eng = _engine(plugins["GatedOscillator"], sa, every, N, TS_OSC, T_OSC, cost=b.AffineCost(1.0, 0.0), tol=1e-12)
    run = _run(eng, u0, p)
    assert np.isfinite(run[2]).all() and np.isfinite(run[3]).all()
    _check_against(run, refs, OSC_MEMBERS, 1e-10, 1e-9, _grad_rtol(sa, 1e-7), f"GatedOscillator {sa}")


@pytest.mark.gpu
@pytest.mark.parametrize("sa,every", SENSEALGS, ids=SA_IDS)
@pytest.mark.parametrize("fam", ["MovingWall", "Gates8", "GatedOscillator"])
def test_shared_p_is_the_sum_of_the_members(plugins, fam, sa, every):
    """shared p: dp is the math.fsum of the per-member dp of the same p given to every member, to 1e-12"""
    inputs, ts, T, cost = {"MovingWall": (wall_inputs, TS_WALL, T_WALL, -1.0), "Gates8": (gate_inputs, TS_GATES, T_GATES, -1.0),
                           "GatedOscillator": (osc_inputs, TS_OSC, T_OSC, 0.0)}[fam]
    u0, p = inputs()
    if fam == "MovingWall":
        u0[0] = p[1, 5] + (u0[0] - p[1])            # the same wall for every member
    ps = p[:, 5].copy()
    runs = []
    for shared in (True, False):
        eng = _engine(plugins[fam], sa, every, N, ts, T, shared_p=shared, cost=b.AffineCost(1.0, cost))
        runs.append(_run(eng, u0, ps if shared else np.tile(ps[:, None], (1, N))))
    (s1, st1, du1, dp1, c1, *_), (s2, st2, du2, dp2, c2, *_) = runs
    assert (st1 == 0).all() and (st2 == 0).all() and np.array_equal(c1, c2) and c1.max() > 0
    assert np.array_equal(s1, s2)
    assert np.allclose(du1, du2, rtol=1e-12, atol=0)
    for q in range(len(ps)):
        ref = math.fsum(dp2[q])
        assert abs(dp1.ravel()[q] - ref) <= 1e-12 * math.fsum(np.abs(dp2[q])), (q, dp1.ravel()[q], ref)


@pytest.mark.gpu
@pytest.mark.parametrize("sa,every", SENSEALGS, ids=SA_IDS)
def test_simultaneous_fire_differentiates_through_the_lowest_condition(plugins, sa, every):
    """CornerWalls started on the diagonal (x0 = y0, vx = vy): both walls fire on the same bits and stop the motion.  The
    event time is a function of either condition; the kernel takes the lowest that fired, x, so
    x(T) = 0 and y(T) = y0 + vy tau with tau = -x0 / vx.  Observed: 3e-14."""
    n = 64
    rng = np.random.default_rng(61)
    a, v = rng.uniform(0.5, 1.5, n), rng.uniform(0.5, 1.5, n)
    u0 = np.stack([a, a, -v, -v])
    T = 3.0
    eng = _engine(plugins["CornerWalls"], sa, every, n, [T], T, shared_p=True)
    saved, status = eng.forward(u0, np.array([0.0]))
    uT = np.asarray(saved)[0].copy()
    dL = np.zeros((1, 4, n)); dL[0, :2] = 2 * (uT[:2] - 0.5)
    du0, _ = eng.reverse(dL)
    counts, _ = eng.event_times()
    flags = eng.event_flags()
    assert (np.asarray(status) == 0).all() and (counts == 1).all() and (flags[0] == -1).all()

    def corner(z):
        tau = -z[0] / z[2]
        return np.sum((np.array([0.0 * z[0], z[1] + z[3] * tau]) - 0.5) ** 2)
    ref = [complex_step_grad(corner, u0[:, i]) for i in range(n)]
    _check_member_grads([np.asarray(du0)[:, i] for i in range(n)], ref, _grad_rtol(sa, 1e-8), f"corner {sa}")


@pytest.mark.gpu
@pytest.mark.parametrize("shared_p", [False, True])
def test_event_capacity_overflow_nans_only_the_overflowed_members(plugins, shared_p):
    """Gates8 with max_events below some members' event counts: those report status 3 and get NaN du0 / dp (shared p: the
    reduced dp is NaN); every other member is bitwise the run with enough capacity."""
    u0, p = gate_inputs()
    if shared_p:
        p = p[:, 7].copy()
    pp = p if shared_p else p
    full = _run(_engine(plugins["Gates8"], "gauss", False, N, TS_GATES, T_GATES, shared_p=shared_p, cost=b.AffineCost(1.0, -1.0)), u0, pp)
    counts = full[4]
    cap = int(np.median(counts))
    over = counts > cap
    assert over.any() and (~over).any() and (full[1] == 0).all()
    eng = _engine(plugins["Gates8"], "gauss", False, N, TS_GATES, T_GATES, shared_p=shared_p, cost=b.AffineCost(1.0, -1.0), max_events=cap)
    saved, status = eng.forward(u0, pp)
    du0, dp = eng.reverse()
    saved, status, du0, dp = (np.asarray(x) for x in (saved, status, du0, dp))
    assert np.array_equal(status, np.where(over, 3, 0))
    assert np.isnan(du0[:, over]).all()
    assert np.array_equal(saved[:, :, ~over], full[0][:, :, ~over]) and np.array_equal(du0[:, ~over], full[2][:, ~over])
    if shared_p:
        assert np.isnan(dp).all()
    else:
        assert np.isnan(dp[:, over]).all() and np.array_equal(dp[:, ~over], full[3][:, ~over])


@pytest.mark.gpu
@pytest.mark.parametrize("sa", ["interpolating", "gauss", "backsolve"])
def test_step_capacity_overflow_nans_only_the_failed_members(sa):
    """plain adaptive Tsit5 (Lotka-Volterra) with max_steps below some members' step counts: those report status 2 and get
    NaN du0 / dp, also when the forward pass was not asked for the status; every other member is bitwise the run with
    enough capacity."""
    n = 96
    rng = np.random.default_rng(71)
    u0 = np.stack([rng.uniform(0.3, 3.0, n), rng.uniform(0.3, 3.0, n)])
    p = np.stack([1.5 + 0.5 * rng.uniform(-1, 1, n), np.ones(n), 3.0 + rng.uniform(-1, 1, n), np.ones(n)])
    ts = np.linspace(0.5, 10.0, 20)
    mk = lambda ms: b.DeviceEnsemble("lv", sa, "tsit5_adaptive", n, ts, (0.0, 10.0), 0.0, shared_p=False, cost=b.AffineCost(1.0, -1.0),
                                     abstol=1e-10, reltol=1e-10, max_steps=ms, ckpt_every_step=sa == "backsolve")
    eng = mk(0)
    s_full, st_full = (np.asarray(x).copy() for x in eng.forward(u0, p))
    du_full, dp_full = (np.asarray(x).copy() for x in eng.reverse())
    nf = np.asarray(eng.step_counts()[0]).copy()
    cap = int(np.median(nf))
    over = nf > cap
    assert (st_full == 0).all() and over.any() and (~over).any()
    eng = mk(cap)
    eng.forward(u0, p, want_status=False)
    du0, dp = (np.asarray(x).copy() for x in eng.reverse())
    assert np.isnan(du0[:, over]).all() and np.isnan(dp[:, over]).all()
    assert np.array_equal(du0[:, ~over], du_full[:, ~over]) and np.array_equal(dp[:, ~over], dp_full[:, ~over])
    saved, status = (np.asarray(x).copy() for x in eng.forward(u0, p))
    assert np.array_equal(status, np.where(over, 2, 0))
    assert np.array_equal(saved[:, :, ~over], s_full[:, :, ~over])
