"""Neural-ODE family (MLP 2->64->64->2, shared weights, BASELINE config C4): InterpolatingAdjoint, fixed-step Tsit5,
batched-state kernels, against the fp64 oracle.  fp64 path: 1e-9; fp32 path: 1e-5 on dp (BASELINE C4's fp32 bound)."""
import os
import sys

import numpy as np
import pytest

pytestmark = pytest.mark.gpu
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))

import scimlsensitivity_jl_b200 as b
from oracle import oracle as O

H = 64
P = H * H + 6 * H + 2


def _weights(seed=1):
    rng = np.random.default_rng(seed)
    W1 = rng.standard_normal((H, 2)) / np.sqrt(2); W2 = rng.standard_normal((H, H)) / np.sqrt(H); W3 = rng.standard_normal((2, H)) / np.sqrt(H)
    b1, b2, b3 = 0.1 * rng.standard_normal(H), 0.1 * rng.standard_normal(H), 0.1 * rng.standard_normal(2)
    return np.concatenate([W1.ravel(order="F"), b1, W2.ravel(order="F"), b2, W3.ravel(order="F"), b3])


def _rel(a, ref):
    return np.abs(np.asarray(a, dtype=np.float64) - ref).max() / max(np.abs(ref).max(), 1e-300)


@pytest.mark.parametrize("dtype,tol_u,tol_p", [("f64", 1e-9, 1e-9), ("f32", 2e-5, 1e-5)])
@pytest.mark.parametrize("cost", ["affine", "explicit"])
@pytest.mark.parametrize("N", [100, 4096])
@pytest.mark.parametrize("sensealg", ["interpolating", "gauss"])
def test_mlp_interpolating_parity(dtype, tol_u, tol_p, cost, N, sensealg):
    """InterpolatingAdjoint, and GaussAdjoint -- the reference's default choice once length(u0) + length(p) > 100
    (src/concrete_solve.jl:291-316; P = 4482 here)."""
    T, dt = 1.5, 0.05
    saveat = np.linspace(0.05, T, 30)
    rng = np.random.default_rng(0)
    u0 = rng.uniform(-2, 2, (2, N)); p = _weights()
    assert p.size == P
    cfg = O.make_cfg("mlp", sensealg, "tsit5_fixed", N, saveat, 0.0, T, dt=dt, cost=("affine", 1.0, -0.5), mlp_hidden=H)
    ref = O.gradient(cfg, saveat, u0, p)
    eng = b.DeviceEnsemble("mlp", sensealg, "tsit5_fixed", N, saveat, (0.0, T), dt, dtype=dtype,
                           cost=b.AffineCost(1.0, -0.5) if cost == "affine" else None)
    saved, status = eng.forward(u0, p)
    assert (status == 0).all()
    assert np.abs(saved - ref["saved"]).max() < (1e-11 if dtype == "f64" else 2e-5)
    du0, dp = eng.reverse(None if cost == "affine" else saved - 0.5)
    assert dp.shape == (P,)
    assert _rel(du0, ref["du0"]) < tol_u
    assert _rel(dp, ref["dp"]) < tol_p
    eng.close()


BLOCKS = {"W1": slice(0, 2 * H), "b1": slice(2 * H, 3 * H), "W2": slice(3 * H, 3 * H + H * H), "b2": slice(3 * H + H * H, 4 * H + H * H),
          "W3": slice(4 * H + H * H, 6 * H + H * H), "b3": slice(6 * H + H * H, P)}


@pytest.mark.parametrize("N", [100, 4096, 12000])
@pytest.mark.parametrize("cost", ["affine", "explicit"])
@pytest.mark.parametrize("sensealg", ["interpolating", "gauss"])
def test_mlp_bf16_tensor_core_path(N, cost, sensealg):
    """dtype = bf16_f32acc (csrc/mlp_tc.cuh): every GEMM-shaped piece of the time loop -- the hidden-layer products of f and
    of its VJP, and ALL parameter-gradient contractions over the members -- runs on wgmma with bf16 operands and fp32 register
    accumulators.  BASELINE C4: <= 2e-2 relative to the fp64 oracle for the bf16 path (observed 1e-3 .. 7e-3)."""
    T, dt = 1.5, 0.05
    saveat = np.linspace(0.05, T, 30)
    rng = np.random.default_rng(0)
    u0 = rng.uniform(-2, 2, (2, N)); p = _weights()
    dL = None if cost == "affine" else rng.standard_normal((30, 2, N))
    # N = 100, 4096: the 32-member layout (mlp_tc.cuh); N = 12000 (> 2 x 132 x 32): the 128-member layout (mlp_tc_wide.cuh)
    cfg = O.make_cfg("mlp", sensealg, "tsit5_fixed", N, saveat, 0.0, T, dt=dt, cost=("affine", 1.0, -0.5) if cost == "affine" else ("explicit",), mlp_hidden=H)
    ref = O.gradient(cfg, saveat, u0, p, dLdu=dL)
    eng = b.DeviceEnsemble("mlp", sensealg, "tsit5_fixed", N, saveat, (0.0, T), dt, dtype="bf16_f32acc",
                           cost=b.AffineCost(1.0, -0.5) if cost == "affine" else None)
    saved, status = eng.forward(u0, p)
    assert (np.asarray(status) == 0).all()
    du0, dp = eng.reverse(dL)
    assert _rel(saved, ref["saved"]) < 1e-2
    assert _rel(du0, ref["du0"]) < 1e-2
    for name, sl in BLOCKS.items():
        assert _rel(np.asarray(dp)[sl], ref["dp"][sl]) < 2e-2, name
    err = np.abs(np.asarray(dp)[BLOCKS["W2"]] - ref["dp"][BLOCKS["W2"]]) / np.abs(ref["dp"][BLOCKS["W2"]]).max()
    assert np.sqrt(np.mean(err ** 2)) < 2e-3                           # typical error: bf16 rounding averaged over the contraction
    # deterministic: same launch, same bits
    du0b, dpb = eng.reverse(dL)
    assert np.array_equal(np.asarray(du0), np.asarray(du0b)) and np.array_equal(np.asarray(dp), np.asarray(dpb))
    eng.close()


def test_mlp_bf16_members_not_a_multiple_of_the_tile():
    """N = 130 = one full 128-member tile + 2: the pad rows of the second tile must contribute nothing to any gradient."""
    N, T, dt = 130, 1.5, 0.05
    saveat = np.linspace(0.05, T, 30)
    rng = np.random.default_rng(3)
    u0 = rng.uniform(-2, 2, (2, N)); p = _weights()
    ref = O.gradient(O.make_cfg("mlp", "interpolating", "tsit5_fixed", N, saveat, 0.0, T, dt=dt, cost=("affine", 1.0, -0.5), mlp_hidden=H), saveat, u0, p)
    eng = b.DeviceEnsemble("mlp", "interpolating", "tsit5_fixed", N, saveat, (0.0, T), dt, dtype="bf16_f32acc", cost=b.AffineCost(1.0, -0.5))
    eng.forward(u0, p)
    du0, dp = eng.reverse()
    assert _rel(du0, ref["du0"]) < 1e-2 and _rel(dp, ref["dp"]) < 2e-2
    eng.close()


def test_mlp_unsupported_combinations_fail_loudly():
    saveat = np.linspace(0.05, 1.5, 30)
    with pytest.raises(b.B200AdjError) as ei:
        b.DeviceEnsemble("mlp", "backsolve", "tsit5_fixed", 64, saveat, (0.0, 1.5), 0.05)
    assert ei.value.code == -2
    with pytest.raises(b.B200AdjError):
        b.DeviceEnsemble("mlp", "interpolating", "tsit5_fixed", 64, saveat, (0.0, 1.5), 0.05, shared_p=False)
