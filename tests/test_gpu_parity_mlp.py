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


def _nsm():
    import torch
    return torch.cuda.get_device_properties(0).multi_processor_count


def _bf16_vs_oracle(N, cost, sensealg, seed=0):
    """dtype = bf16_f32acc against the fp64 oracle at BASELINE C4's bounds, plus same-launch determinism; -> (dp, oracle dp)"""
    T, dt = 1.5, 0.05
    saveat = np.linspace(0.05, T, 30)
    rng = np.random.default_rng(seed)
    u0 = rng.uniform(-2, 2, (2, N)); p = _weights()
    dL = None if cost == "affine" else rng.standard_normal((30, 2, N))
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
    # deterministic: same launch, same bits
    du0b, dpb = eng.reverse(dL)
    assert np.array_equal(np.asarray(du0), np.asarray(du0b)) and np.array_equal(np.asarray(dp), np.asarray(dpb))
    eng.close()
    return np.asarray(dp), ref["dp"]


@pytest.mark.parametrize("N", [100, 4096, 12000])
@pytest.mark.parametrize("cost", ["affine", "explicit"])
@pytest.mark.parametrize("sensealg", ["interpolating", "gauss"])
def test_mlp_bf16_tensor_core_path(N, cost, sensealg):
    """dtype = bf16_f32acc (csrc/mlp_tc.cuh): every GEMM-shaped piece of the time loop -- the hidden-layer products of f and
    of its VJP, and ALL parameter-gradient contractions over the members -- runs on wgmma with bf16 operands and fp32 register
    accumulators.  BASELINE C4: <= 2e-2 relative to the fp64 oracle for the bf16 path (observed 1e-3 .. 7e-3)."""
    # N = 100, 4096: the 32-member layout (mlp_tc.cuh); N = 12000 (> 64 x 132 SMs): the 128-member layout (mlp_tc_wide.cuh)
    dp, ref_dp = _bf16_vs_oracle(N, cost, sensealg)
    err = np.abs(dp[BLOCKS["W2"]] - ref_dp[BLOCKS["W2"]]) / np.abs(ref_dp[BLOCKS["W2"]]).max()
    assert np.sqrt(np.mean(err ** 2)) < 2e-3                           # typical error: bf16 rounding averaged over the contraction


# The host runs the 32-member layout while ceil(N / 32) <= 2 x n_SM, i.e. up to N = 64 n_SM, and the 128-member layout beyond.
LAYOUT_SIZES = {"1": lambda nsm: 1, "33": lambda nsm: 33, "last_narrow": lambda nsm: 64 * nsm,
                "first_wide": lambda nsm: 64 * nsm + 1, "wide_last_tile_127": lambda nsm: 64 * nsm + 127}


@pytest.mark.parametrize("size", list(LAYOUT_SIZES))
@pytest.mark.parametrize("sensealg", ["interpolating", "gauss"])
def test_mlp_bf16_layout_boundaries(size, sensealg):
    """Both sides of the narrow -> wide switch, which follows the device's SM count: a single member, one full narrow CTA + 1,
    the largest narrow size, the first wide size (its last 128-member tile holds ONE live member) and a last tile of 127."""
    _bf16_vs_oracle(LAYOUT_SIZES[size](_nsm()), "affine", sensealg, seed=5)


@pytest.mark.parametrize("layout", ["narrow", "wide"])
@pytest.mark.parametrize("sensealg", ["interpolating", "gauss"])
def test_mlp_bf16_member_permutation(layout, sensealg):
    """A member's trajectory and adjoint depend only on its own MMA row: moving every member to another CTA and another row
    of it (a cyclic shift) leaves saved and du0 bit-identical; dp, a sum over CTAs in another order, agrees to 1e-5."""
    nsm = _nsm()
    N, tile = (64 * nsm - 45, 32) if layout == "narrow" else (64 * nsm + 77, 128)     # both with a ragged last tile
    shift = 1061                                               # 8 x 128 + 37
    order = np.roll(np.arange(N), shift)                       # position q runs member order[q]; member m sits at (m + shift) % N
    pos = (np.arange(N) + shift) % N
    assert ((pos // tile) != (np.arange(N) // tile)).all() and ((pos % tile) != (np.arange(N) % tile)).all()
    T, dt = 1.5, 0.05
    saveat = np.linspace(0.05, T, 30)
    rng = np.random.default_rng(6)
    u0 = rng.uniform(-2, 2, (2, N)); p = _weights()
    out = []
    for perm in (np.arange(N), order):
        eng = b.DeviceEnsemble("mlp", sensealg, "tsit5_fixed", N, saveat, (0.0, T), dt, dtype="bf16_f32acc", cost=b.AffineCost(1.0, -0.5))
        saved, _ = eng.forward(u0[:, perm], p)
        du0, dp = eng.reverse()
        saved, du0 = np.array(saved), np.array(du0)
        saved[..., perm] = saved.copy(); du0[:, perm] = du0.copy()                # back to member order
        out.append((saved, du0, np.array(dp)))
        eng.close()
    (s0, u0_, p0), (s1, u1, p1) = out
    assert np.array_equal(s0, s1)
    assert np.array_equal(u0_, u1)
    assert _rel(p1, p0) < 1e-5


def test_mlp_bf16_members_not_a_multiple_of_the_tile():
    """N = 64 n_SM + 2, among the first sizes of the 128-member layout: the last tile holds 2 live members and 126 pad rows,
    which must contribute nothing to any gradient."""
    N, T, dt = 64 * _nsm() + 2, 1.5, 0.05
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
