"""The support matrix of the C ABI as a table: which (family, stepper, dtype, sensealg, checkpointing, event, callback)
combinations each entry point refuses, and with which status code.  One accepted configuration per execution path
(fixed-grid Tsit5, dense per-member Tsit5, Rosenbrock23, SDE, MLP) runs a forward and a reverse pass."""
import ctypes as C
import os

import numpy as np
import pytest

pytestmark = pytest.mark.gpu

from scimlsensitivity_jl_b200 import _lib as L

OK, INVALID, UNSUPPORTED, NO_DEVICE, STATE = 0, -1, -2, -3, -5
DIMS = {"lv": (2, 4), "lorenz": (3, 3), "robertson": (3, 3), "sde_lv": (2, 6), "sde_linear": (2, 2), "ball": (2, 2),
        "relax": (1, 2), "mlp": (2, 4482)}
N = 4


def _cfg(family="lv", sensealg="gauss", stepper="tsit5_fixed", dtype="f64", saveat=(0.5, 1.0), t1=1.0, dt=0.1, **kw):
    c = L.Cfg()
    c.rhs_family = L.FAM.get(family, family) if isinstance(family, str) else family
    c.d, c.P = DIMS.get(family, (2, 4))
    c.sensealg = L.SA.get(sensealg, sensealg) if isinstance(sensealg, str) else sensealg
    c.stepper, c.dtype = L.ST[stepper], L.DTYPE[dtype]
    c.N, c.t0, c.t1, c.dt = N, 0.0, t1, dt
    c.abstol, c.reltol, c.quad_abstol, c.quad_reltol = 1e-8, 1e-6, 1e-8, 1e-6
    c.shared_p, c.cost_kind, c.cost_a, c.cost_b, c.mlp_hidden = 1, L.COST["affine"], 1.0, 0.0, 64
    c._keep = np.ascontiguousarray(saveat, dtype=np.float64)
    c.K = len(c._keep)
    c.saveat = c._keep.ctypes.data_as(C.POINTER(C.c_double)) if c.K else None
    for k, v in kw.items():
        setattr(c, k, v)
    return c


class _H:
    """A raw handle: every call returns the status code."""

    def __init__(self, cfg):
        self.lib, self.cfg, self.h = L.load(), cfg, C.c_void_p()
        self.rc = self.lib.b200adj_create(C.byref(cfg), C.byref(self.h))

    def __getattr__(self, name):
        fn = getattr(self.lib, "b200adj_" + name)
        return lambda *a: fn(self.h, *a)

    def arrays(self):
        c = self.cfg
        real = np.float64 if c.dtype == L.DTYPE["f64"] else np.float32
        u0 = np.full((c.d, N), 0.5, dtype=real)
        p = np.full(c.P, 0.01 if c.rhs_family == L.FAM["mlp"] else 0.5, dtype=real)
        return u0, p, np.zeros((c.d, N), dtype=real), np.zeros(c.P, dtype=real)

    def run(self):
        u0, p, du0, dp = self.arrays()
        rc = self.forward(u0.ctypes.data, p.ctypes.data, None, None, None)
        return rc if rc else self.reverse(None, du0.ctypes.data, dp.ctypes.data)

    def close(self):
        if self.h:
            self.lib.b200adj_destroy(self.h)
            self.h = C.c_void_p()


def _d(x):
    x = np.ascontiguousarray(x, dtype=np.float64)
    return x, x.ctypes.data


def _handle(**kw):
    h = _H(_cfg(**kw))
    assert h.rc == OK, L.load().b200adj_last_error(None)
    return h


# configurations per execution path
FIXED = dict()
DENSE = dict(saveat=(0.25, 1.0))                                   # off the dt grid: the dense per-member framework
T5A = dict(stepper="tsit5_adaptive", saveat=(0.25, 1.0))
ROS = dict(stepper="rosenbrock23", saveat=(0.25, 1.0))
SDE = dict(family="sde_lv", stepper="em", sensealg="backsolve")
MLP = dict(family="mlp", dt=0.25)

CREATE = [
    (dict(device=-1, family=42), NO_DEVICE),
    (dict(family=42), UNSUPPORTED),
    (dict(family="mlp", mlp_hidden=32), UNSUPPORTED),
    (dict(d=3), INVALID),
    (dict(DENSE, checkpoint_every=4), UNSUPPORTED),
    (dict(N=0), INVALID),
    (dict(t1=0.0), INVALID),
    (dict(dtype="f32", sensealg="quadrature"), UNSUPPORTED),
    (dict(family="robertson", dtype="f32"), UNSUPPORTED),
    (dict(dtype="bf16_f32acc"), UNSUPPORTED),
    (dict(ROS, dtype="f32"), UNSUPPORTED),
    (dict(MLP, stepper="rosenbrock23"), UNSUPPORTED),
    (dict(MLP, sensealg="quadrature"), UNSUPPORTED),
    (dict(MLP, sensealg="backsolve"), UNSUPPORTED),
    (dict(MLP, shared_p=0), UNSUPPORTED),
    (dict(cost_kind=5), INVALID),
    (dict(SDE, family="lv"), INVALID),
    (dict(SDE, sensealg="gauss"), UNSUPPORTED),
    (dict(SDE, sensealg="quadrature"), UNSUPPORTED),
    (dict(family="sde_linear"), INVALID),
    (dict(sensealg=7), INVALID),
    (dict(dtype="f32", sensealg="gauss_kronrod"), UNSUPPORTED),
    (dict(ROS, abstol=0.0), INVALID),
    (dict(T5A, reltol=0.0), INVALID),
    (dict(family="ball"), UNSUPPORTED),
    (dict(family="relax"), UNSUPPORTED),
    (dict(T5A, saveat=(0.5, 0.25)), INVALID),
    (dict(ROS, saveat=(0.5, 1.5)), INVALID),
    (dict(saveat=(0.5,), dt=0.3), UNSUPPORTED),                     # dense framework, (t1 - t0) not a whole number of steps
    (dict(T5A, block_threads=512), INVALID),
    (dict(saveat=(), dt=0.3), UNSUPPORTED),                         # fixed grid, (t1 - t0) not a whole number of steps
    (dict(saveat=(0.5, 0.5)), UNSUPPORTED),
    (dict(saveat=(0.5, 0.2)), INVALID),
    (dict(block_threads=48), INVALID),
    (dict(checkpoint_every=4, sensealg="backsolve"), UNSUPPORTED),
    (dict(SDE, checkpoint_every=4), UNSUPPORTED),
    (dict(MLP, checkpoint_every=2), UNSUPPORTED),
    (dict(family="lorenz", checkpoint_every=20, block_threads=512, dt=0.01), INVALID),   # checkpoint tile > 160 KB
    # several faults at once: the order of the checks decides the code
    (dict(MLP, sensealg="backsolve", cost_kind=5), UNSUPPORTED),
    (dict(MLP, sensealg=7), UNSUPPORTED),
    (dict(dtype="f32", sensealg="quadrature", cost_kind=5), UNSUPPORTED),
    (dict(dtype="f32", sensealg="gauss_kronrod", cost_kind=5), INVALID),
    (dict(SDE, sensealg="gauss", cost_kind=5), INVALID),
    (dict(SDE, sensealg=7), UNSUPPORTED),
    (dict(sensealg=7, checkpoint_every=4), INVALID),
    (dict(checkpoint_every=4, sensealg="backsolve", block_threads=48), INVALID),
    (dict(checkpoint_every=4, sensealg="backsolve", saveat=(0.5, 0.2)), INVALID),
    (dict(checkpoint_every=4, sensealg="backsolve", saveat=(0.5, 0.5)), UNSUPPORTED),
    (dict(MLP, checkpoint_every=2, block_threads=48), INVALID),
    (dict(SDE, checkpoint_every=4, block_threads=48), INVALID),
    (dict(family="lorenz", checkpoint_every=20, block_threads=512, dt=0.01, sensealg="backsolve"), UNSUPPORTED),
]


@pytest.mark.parametrize("kw,code", CREATE)
def test_create(kw, code):
    h = _H(_cfg(**kw))
    try:
        assert h.rc == code, (kw, L.load().b200adj_last_error(None))
    finally:
        h.close()


def test_create_null_cfg():
    assert L.load().b200adj_create(None, C.byref(C.c_void_p())) == INVALID


ACCEPTED = [FIXED, dict(FIXED, sensealg="quadrature"), dict(FIXED, dtype="f32", family="lorenz", sensealg="backsolve"),
            dict(FIXED, checkpoint_every=4, sensealg="interpolating"), DENSE, T5A, dict(T5A, sensealg="gauss_kronrod"),
            dict(T5A, family="ball"), ROS, dict(ROS, sensealg="quadrature"), SDE, dict(SDE, sensealg="interpolating"),
            MLP, dict(MLP, dtype="f32"), dict(MLP, dtype="bf16_f32acc", sensealg="interpolating")]


@pytest.mark.parametrize("kw", ACCEPTED)
def test_accepted_paths_run(kw):
    h = _handle(**kw)
    try:
        assert h.run() == OK, h.last_error()
    finally:
        h.close()


def _ropt(h, sensealg, cost="affine", t=None):
    sa = L.SA.get(sensealg, sensealg) if isinstance(sensealg, str) else sensealg
    ck = L.COST.get(cost, cost) if isinstance(cost, str) else cost
    if t is None:
        return h.set_reverse_options(sa, ck, 1.0, 0.0, 0, -1, None)
    t, tp = _d(t)
    return h.set_reverse_options(sa, ck, 1.0, 0.0, 0, len(t), tp if len(t) else None)


REVERSE_OPTIONS = [
    (FIXED, dict(sensealg=9), INVALID),
    (FIXED, dict(sensealg="gauss", cost=3), INVALID),
    (SDE, dict(sensealg="gauss_kronrod"), UNSUPPORTED),
    (MLP, dict(sensealg="gauss_kronrod"), UNSUPPORTED),
    (dict(FIXED, dtype="f32"), dict(sensealg="gauss_kronrod"), UNSUPPORTED),
    (dict(FIXED, checkpoint_every=4), dict(sensealg="backsolve"), UNSUPPORTED),
    (dict(FIXED, checkpoint_every=4), dict(sensealg="quadrature"), UNSUPPORTED),
    (SDE, dict(sensealg="gauss"), UNSUPPORTED),
    (MLP, dict(sensealg="backsolve"), UNSUPPORTED),
    (MLP, dict(sensealg="quadrature"), UNSUPPORTED),
    (dict(FIXED, dtype="f32"), dict(sensealg="quadrature"), UNSUPPORTED),
    (FIXED, dict(sensealg="gauss", t=(0.25,)), UNSUPPORTED),         # off the dt grid
    (FIXED, dict(sensealg="gauss", t=(0.5, 0.5)), UNSUPPORTED),
    (T5A, dict(sensealg="gauss", t=(0.5, 1.5)), INVALID),
    (DENSE, dict(sensealg="gauss", t=(0.5, 0.25)), INVALID),
    (ROS, dict(sensealg="gauss", t=(-0.5,)), INVALID),
    # accepted
    (FIXED, dict(sensealg="quadrature", t=(0.2, 0.6)), OK),
    (FIXED, dict(sensealg="gauss_kronrod"), OK),
    (DENSE, dict(sensealg="quadrature", t=(0.15, 0.35)), OK),
    (T5A, dict(sensealg="backsolve", cost="explicit", t=(0.3,)), OK),
    (ROS, dict(sensealg="gauss_kronrod"), OK),
    (SDE, dict(sensealg="interpolating"), OK),
    (MLP, dict(sensealg="interpolating"), OK),
]


@pytest.mark.parametrize("kw,args,code", REVERSE_OPTIONS)
def test_set_reverse_options(kw, args, code):
    h = _handle(**kw)
    try:
        assert _ropt(h, **args) == code, h.last_error()
        if code == OK and args.get("cost") != "explicit":
            assert h.run() == OK, h.last_error()
    finally:
        h.close()


def test_set_reverse_options_null_save_times():
    for kw in (FIXED, T5A, ROS):
        h = _handle(**kw)
        try:
            assert h.set_reverse_options(L.SA["gauss"], L.COST["affine"], 1.0, 0.0, 0, 2, None) == INVALID
        finally:
            h.close()


def _events(h, E=1, times=None, pshift=False):
    d, P = h.cfg.d, h.cfg.P
    E = len(times) if times is not None else E
    t, tp = _d(times if times is not None else np.linspace(0.0, 1.0, E + 2)[1:-1] if E > 0 else [0.0])
    s, sp = _d(np.ones((max(E, 1), d)))
    c, cp = _d(np.zeros((max(E, 1), d)))
    ps, psp = _d(np.ones((max(E, 1), P)))
    pc, pcp = _d(np.zeros((max(E, 1), P)))
    return h.set_events(E, tp, sp, cp, psp if pshift else None, pcp if pshift else None)


def _callback(h, enabled=1, idx=0, max_events=4):
    return h.set_continuous_callback(enabled, idx, 0.0, -1, None, None, -1, 0, 1.0, max_events)


EVENTS = [
    (FIXED, dict(E=-1), INVALID),
    (ROS, dict(), UNSUPPORTED),
    (SDE, dict(), UNSUPPORTED),
    (dict(FIXED, dtype="f32"), dict(), UNSUPPORTED),
    (dict(MLP, dtype="bf16_f32acc"), dict(), UNSUPPORTED),
    (MLP, dict(pshift=True), UNSUPPORTED),
    (dict(FIXED, checkpoint_every=4), dict(), UNSUPPORTED),
    (FIXED, dict(times=(0.35,)), UNSUPPORTED),                      # off the dt grid
    (FIXED, dict(times=(0.5, 0.5)), INVALID),
    (dict(FIXED, sensealg="quadrature"), dict(), UNSUPPORTED),
    (dict(T5A, sensealg="quadrature"), dict(), UNSUPPORTED),
    (T5A, dict(times=(0.5, 0.3)), INVALID),
    (T5A, dict(times=(1.0,)), INVALID),
    # accepted
    (FIXED, dict(times=(0.5,), pshift=True), OK),
    (DENSE, dict(times=(0.35,)), OK),
    (T5A, dict(times=(0.35,), pshift=True), OK),
    (MLP, dict(times=(0.5,)), OK),
    (ROS, dict(E=0), OK),
]


@pytest.mark.parametrize("kw,args,code", EVENTS)
def test_set_events(kw, args, code):
    h = _handle(**kw)
    try:
        assert _events(h, **args) == code, h.last_error()
        if code == OK:
            assert h.run() == OK, h.last_error()
    finally:
        h.close()


def test_set_events_with_a_continuous_callback():
    h = _handle(**dict(T5A, family="ball"))
    try:
        assert _callback(h) == OK
        assert _events(h) == UNSUPPORTED
    finally:
        h.close()


def _shift(h, comp=(0,), param=(1,), coef=(1.0,), null_param=False):
    a, b, c = (np.ascontiguousarray(comp, dtype=np.int32), np.ascontiguousarray(param, dtype=np.int32),
               np.ascontiguousarray(coef, dtype=np.float64))
    return h.set_event_param_shift(a.ctypes.data, None if null_param else b.ctypes.data, c.ctypes.data)


PARAM_SHIFT = [
    (T5A, None, dict(), STATE),
    (T5A, dict(times=(0.35,)), dict(null_param=True), INVALID),
    (FIXED, dict(times=(0.5,)), dict(), UNSUPPORTED),
    (MLP, dict(times=(0.5,)), dict(), UNSUPPORTED),
    (T5A, dict(times=(0.35,)), dict(comp=(5,)), INVALID),
    (T5A, dict(times=(0.35,)), dict(param=(9,)), INVALID),
    (T5A, dict(times=(0.35,)), dict(), OK),
    (DENSE, dict(times=(0.35,)), dict(), OK),
]


@pytest.mark.parametrize("kw,ev,args,code", PARAM_SHIFT)
def test_set_event_param_shift(kw, ev, args, code):
    h = _handle(**kw)
    try:
        if ev is not None:
            assert _events(h, **ev) == OK, h.last_error()
        assert _shift(h, **args) == code, h.last_error()
        if ev is not None:
            assert h.set_event_param_shift(None, None, None) == OK
        if code == OK:
            assert _shift(h, **args) == OK and h.run() == OK, h.last_error()
    finally:
        h.close()


CONT_COST = [(ROS, UNSUPPORTED), (SDE, UNSUPPORTED), (MLP, UNSUPPORTED), (FIXED, OK), (DENSE, OK), (T5A, OK),
             (dict(FIXED, checkpoint_every=4), OK)]


@pytest.mark.parametrize("kw,code", CONT_COST)
def test_set_continuous_cost(kw, code):
    h = _handle(**kw)
    try:
        assert h.set_continuous_cost(1, 1.0, 0.5) == code, h.last_error()
        assert h.set_continuous_cost(0, 0.0, 0.0) == OK
        if code == OK:
            assert h.set_continuous_cost(1, 1.0, 0.5) == OK and h.run() == OK, h.last_error()
    finally:
        h.close()


def test_continuous_cost_on_fp32_is_refused_by_the_reverse_pass():
    h = _handle(**dict(FIXED, dtype="f32"))
    try:
        assert h.set_continuous_cost(1, 1.0, 0.5) == OK
        assert h.run() == UNSUPPORTED
    finally:
        h.close()


def test_set_cost_family():
    for kw, which, dgdp, code in [(MLP, 0, True, UNSUPPORTED), (ROS, 1, False, UNSUPPORTED), (FIXED, 0, True, OK),
                                  (T5A, 1, True, OK)]:
        h = _handle(**kw)
        try:
            e, ep = _d(np.ones(8))
            assert h.set_cost_family(which, None, None, None, ep if dgdp else None) == code, (kw, h.last_error())
        finally:
            h.close()


CALLBACK = [
    (FIXED, dict(), UNSUPPORTED),
    (DENSE, dict(), UNSUPPORTED),
    (ROS, dict(), UNSUPPORTED),
    (dict(T5A, family="ball", sensealg="quadrature"), dict(), UNSUPPORTED),
    (dict(T5A, family="ball"), dict(idx=2), INVALID),
    (dict(T5A, family="ball"), dict(max_events=0), INVALID),
    (FIXED, dict(enabled=0), OK),
    (dict(T5A, family="ball"), dict(), OK),
]


@pytest.mark.parametrize("kw,args,code", CALLBACK)
def test_set_continuous_callback(kw, args, code):
    h = _handle(**kw)
    try:
        assert _callback(h, **args) == code, h.last_error()
        if code == OK:
            assert h.run() == OK, h.last_error()
    finally:
        h.close()


def test_continuous_callback_with_preset_events_and_quadrature():
    h = _handle(**T5A)
    try:
        assert _events(h) == OK
        assert _callback(h) == UNSUPPORTED                           # not together with preset-time events
        assert _events(h, E=0) == OK and _callback(h) == OK
        assert _ropt(h, "quadrature") == UNSUPPORTED                  # no callback support in QuadratureAdjoint
    finally:
        h.close()


STEP_COUNTS = [(FIXED, UNSUPPORTED), (SDE, UNSUPPORTED), (MLP, UNSUPPORTED), (DENSE, OK), (T5A, OK), (ROS, OK)]


@pytest.mark.parametrize("kw,code", STEP_COUNTS)
def test_get_step_counts(kw, code):
    h = _handle(**kw)
    try:
        if code == OK:
            assert h.run() == OK, h.last_error()
        f, r = np.zeros(N, dtype=np.int32), np.zeros(N, dtype=np.int32)
        assert h.get_step_counts(f.ctypes.data, r.ctypes.data) == code, h.last_error()
        if code == OK:
            assert (f > 0).all()
    finally:
        h.close()


@pytest.fixture(scope="module")
def vanderpol():
    """The van der Pol plug-in (examples/vanderpol_family.cuh: d = 2, P = 2, no Jacobian, so no Rosenbrock23 kernels)."""
    import scimlsensitivity_jl_b200 as b
    root = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
    so = os.path.join(root, "examples", "libb200fam_vanderpol.so")
    if not os.path.exists(so):
        so = b.build_family_plugin(os.path.join(root, "examples", "vanderpol_family.cuh"), "VanDerPol", "vanderpol", out=so)
    return b.register_family(so)[0]


def test_plugin_family(vanderpol):
    vdp = dict(family=vanderpol)
    DIMS[vanderpol] = (2, 2)
    assert _H(_cfg(**vdp, d=3)).rc == INVALID
    assert _H(_cfg(**vdp, dtype="f32")).rc == UNSUPPORTED
    for kw, code in [(vdp, OK), (dict(vdp, sensealg="quadrature"), OK), (dict(T5A, **vdp), OK), (dict(ROS, **vdp), UNSUPPORTED)]:
        h = _handle(**kw)
        try:
            assert h.run() == code, (kw, h.last_error())
            if code == OK:
                assert _ropt(h, "gauss_kronrod") == OK and h.run() == OK, h.last_error()
        finally:
            h.close()
