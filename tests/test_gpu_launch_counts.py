"""Kernel launches per forward and per reverse pass (b200adj_launch_count), one small configuration per execution path and
sensealg group.  The counts are part of each path's cost: a launcher that loses or gains a launch changes it."""
import numpy as np
import pytest

pytestmark = pytest.mark.gpu

from scimlsensitivity_jl_b200 import _lib as L
from test_gpu_support_matrix import DENSE, FIXED, MLP, OK, ROS, SDE, T5A, _callback, _d, _events, _handle

# (configuration, forward launches, reverse launches)
COUNTS = [
    (FIXED, 1, 1),
    (dict(FIXED, sensealg="interpolating"), 1, 1),
    (dict(FIXED, sensealg="backsolve", cost_kind=L.COST["explicit"]), 1, 1),
    (dict(FIXED, sensealg="gauss_kronrod"), 1, 1),
    (dict(FIXED, sensealg="quadrature"), 1, 2),
    (dict(FIXED, shared_p=0, sensealg="quadrature"), 1, 2),
    (dict(FIXED, checkpoint_every=4, sensealg="interpolating"), 1, 1),
    (dict(FIXED, dtype="f32", family="lorenz"), 1, 1),
    (dict(FIXED, dtype="f32", family="lorenz", sensealg="backsolve", shared_p=0), 1, 1),
    (DENSE, 1, 1),
    (dict(DENSE, sensealg="quadrature"), 1, 2),
    (T5A, 1, 1),
    (dict(T5A, sensealg="gauss_kronrod", shared_p=0), 1, 1),
    (dict(T5A, sensealg="quadrature"), 1, 2),
    (ROS, 1, 1),
    (dict(ROS, sensealg="backsolve", shared_p=0), 1, 1),
    (dict(ROS, sensealg="quadrature"), 1, 3),
    (SDE, 1, 1),
    (dict(SDE, sensealg="interpolating", stepper="euler_heun"), 1, 1),
    (MLP, 1, 2),
    (dict(MLP, sensealg="interpolating", dtype="f32"), 1, 2),
    (dict(MLP, dtype="bf16_f32acc"), 1, 2),
]


def _counts(h):
    c = h.cfg
    real = np.float64 if c.dtype == L.DTYPE["f64"] else np.float32
    n = c.N
    u0 = np.full((c.d, n), 0.5, dtype=real)
    p = np.full(c.P if c.shared_p else (c.P, n), 0.01 if c.rhs_family == L.FAM["mlp"] else 0.5, dtype=real)
    du0, dp = np.zeros_like(u0), np.zeros_like(p)
    dL = np.ones((c.K, c.d, n), dtype=real)
    l0 = h.launch_count()
    assert h.forward(u0.ctypes.data, p.ctypes.data, None, None, None) == OK, h.last_error()
    l1 = h.launch_count()
    assert h.reverse(dL.ctypes.data, du0.ctypes.data, dp.ctypes.data) == OK, h.last_error()
    return l1 - l0, h.launch_count() - l1


@pytest.mark.parametrize("kw,fwd,rev", COUNTS)
def test_launch_counts(kw, fwd, rev):
    h = _handle(**kw)
    try:
        assert _counts(h) == (fwd, rev)
    finally:
        h.close()


@pytest.mark.parametrize("kw", [dict(FIXED, times=(0.5,)), dict(DENSE, times=(0.35,))])
def test_launch_counts_preset_events(kw):
    kw = dict(kw)
    times = kw.pop("times")
    h = _handle(**kw)
    try:
        assert _events(h, times=times) == OK, h.last_error()
        assert _counts(h) == (1, 1)
    finally:
        h.close()


@pytest.mark.parametrize("kw", [FIXED, T5A])
def test_launch_counts_continuous_cost(kw):
    h = _handle(**kw)
    try:
        assert h.set_continuous_cost(1, 1.0, 0.5) == OK, h.last_error()
        assert _counts(h) == (1, 1)
    finally:
        h.close()


def test_launch_counts_continuous_callback():
    h = _handle(**dict(T5A, family="ball"))
    try:
        assert _callback(h) == OK, h.last_error()
        assert _counts(h) == (1, 1)
    finally:
        h.close()


def test_launch_counts_bf16_wide_layout():
    """past 2 CTAs of 32 members per SM the tensor-core path switches to 128-member CTAs: still one launch each way plus
    the dp reduction"""
    h = _handle(**dict(MLP, dtype="bf16_f32acc", N=2 * 132 * 32 + 128))
    try:
        assert _counts(h) == (1, 2)
    finally:
        h.close()


@pytest.mark.parametrize("kw", [FIXED, dict(FIXED, dtype="f32", family="lorenz"), T5A, ROS, SDE])
def test_launch_counts_parameter_cost(kw):
    """a parameter part of the cost (dgdp) is one more launch after the reverse kernels"""
    h = _handle(**kw)
    try:
        e, ep = _d(np.ones(8))
        assert h.set_cost_family(0, None, None, None, ep) == OK, h.last_error()
        assert _counts(h) == (1, 2)
    finally:
        h.close()
