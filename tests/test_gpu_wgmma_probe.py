"""The tensor-core building blocks of the bf16 neural-ODE kernels (csrc/wgmma.cuh, csrc/mlp_tc.cuh, csrc/mlp_tc_wide.cuh),
one CTA at a time, through tests/csrc/wgmma_probe.cu: the production device functions wrapped in one-CTA kernels.

* GEMM plumbing, bit for bit: bf16 integers in [-8, 8] times one power of two per A row and per B column make every
  product of a (row, col) share one scale, so the fp32 accumulation is exact and numpy's fp64 product is THE answer.
  This pins the shared-memory descriptors, the transpose flags, the accumulator-fragment staging and the
  fragment-to-parameter store of the gradient GEMMs.
* One adjoint stage (forward + VJP + gradient GEMMs) against an fp64 emulation that rounds to bf16 where the kernels do;
  the tolerance is derived from the spread that tanh.approx.f32's 2^-11 relative error causes in that emulation.
* Exact relations of the stage: the quadrature weight wt is only a power-of-two scale, and dead members contribute nothing.
"""
import ctypes as C
import os
import subprocess

import numpy as np
import pytest

from scimlsensitivity_jl_b200 import _lib

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
CSRC = os.path.join(ROOT, "scimlsensitivity.jl_b200", "csrc")
PROBE = os.path.join(ROOT, "tests", "csrc", "wgmma_probe.cu")

H, P = 64, 4482
OW1, OB1, OW2, OB2, OW3, OB3 = 0, 128, 192, 4288, 4352, 4480
BLOCKS = {"W1": slice(OW1, OB1), "b1": slice(OB1, OW2), "W2": slice(OW2, OB2), "b2": slice(OB2, OW3), "W3": slice(OW3, OB3), "b3": slice(OB3, P)}
LAYOUTS = {"narrow": 0, "wide": 1}          # 32 members per CTA (TcSmem) / 128 members per CTA (TcwSmem)
ROWS = {"narrow": 64, "wide": 128}          # rows of the member MMAs (narrow: 32 members + 32 pad rows)
MEMBERS = {"narrow": 32, "wide": 128}       # members of one CTA = K of the gradient GEMMs
TA_F, TB_F, TC_F = 128, 80, 16


@pytest.fixture(scope="session")
def probe_so(tmp_path_factory):
    """wgmma_probe.cu built with the library's own nvcc flags, once per session, outside the source tree."""
    so = str(tmp_path_factory.mktemp("wgmma_probe") / "libwgmma_probe.so")
    cmd = [_lib.nvcc_path(), "-gencode", "arch=compute_90a,code=sm_90a", "-O3", "-std=c++17", "-I", CSRC,
           "-Xcompiler", "-fPIC", "-shared", PROBE, "-o", so]
    res = subprocess.run(cmd, capture_output=True, text=True)
    assert res.returncode == 0, res.stdout[-3000:] + res.stderr[-3000:]
    return so


def test_probe_compiles_for_sm90a(probe_so):
    """No GPU needed: a header change that breaks the probes fails here."""
    assert os.path.getsize(probe_so) > 0
    lib = C.CDLL(probe_so)
    for name in ("probe_member_gemm", "probe_grad_gemm", "probe_stage", "probe_tanh_approx", "probe_pack_bf16"):
        getattr(lib, name)


@pytest.fixture(scope="module")
def probe(probe_so):
    lib = C.CDLL(probe_so)
    vp = C.c_void_p
    lib.probe_member_gemm.argtypes = [C.c_int, C.c_int, vp, vp, C.c_int, vp]
    lib.probe_grad_gemm.argtypes = [C.c_int, vp, C.c_int, vp, vp, vp, vp, vp]
    lib.probe_stage.argtypes = [C.c_int, vp, vp, vp, vp, C.c_float, vp, vp, vp]
    for f in (lib.probe_member_gemm, lib.probe_grad_gemm, lib.probe_stage):
        f.restype = C.c_int
    return lib


def _dev(x, dtype=None):
    import torch
    return torch.tensor(np.ascontiguousarray(x), dtype=dtype or torch.float32, device="cuda")


def _host(t):
    return t.cpu().numpy().astype(np.float64)


def _check(rc):
    assert rc == 0, f"probe launch failed: cudaError {rc}"


def _ints(rng, shape):
    return rng.integers(-8, 9, size=shape).astype(np.float64)


def _pow2(rng, n):
    return np.exp2(rng.integers(-12, 13, size=n)).astype(np.float64)


def _weights(seed=1):
    """The layout [W1 | b1 | W2 | b2 | W3 | b3], every block column-major (as test_gpu_parity_mlp._weights)."""
    rng = np.random.default_rng(seed)
    W1 = rng.standard_normal((H, 2)) / np.sqrt(2); W2 = rng.standard_normal((H, H)) / np.sqrt(H); W3 = rng.standard_normal((2, H)) / np.sqrt(H)
    b1, b2, b3 = 0.1 * rng.standard_normal(H), 0.1 * rng.standard_normal(H), 0.1 * rng.standard_normal(2)
    return np.concatenate([W1.ravel(order="F"), b1, W2.ravel(order="F"), b2, W3.ravel(order="F"), b3])


def _unpack(p):
    """-> W1[j][c], b1, W2[i][j], b2, W3[c][n], b3 out of the flat layout"""
    return (p[BLOCKS["W1"]].reshape(2, H).T, p[BLOCKS["b1"]], p[BLOCKS["W2"]].reshape(H, H).T, p[BLOCKS["b2"]],
            p[BLOCKS["W3"]].reshape(H, 2).T, p[BLOCKS["b3"]])


def _pack(dW1, db1, dW2, db2, dW3, db3):
    return np.concatenate([dW1.ravel(order="F"), db1, dW2.ravel(order="F"), db2, dW3.ravel(order="F"), db3])


def _assert_exact_in_fp32(x):
    assert np.array_equal(x.astype(np.float32).astype(np.float64), x), "test construction: reference not exact in fp32"


# ------------------------------------------------------------------------------------------------------------------------
# member GEMMs: D = A W2' (the forward's Z2 = H1 W2', tile TB) and D = A W2 (the VJP's dH1 = dZ2 W2, tile TA), both tiles
# against both weight tiles


@pytest.mark.gpu
@pytest.mark.parametrize("w2t", [0, 1], ids=["W2", "W2T"])
@pytest.mark.parametrize("tile_f", [TB_F, TA_F], ids=["TB", "TA"])
@pytest.mark.parametrize("layout", list(LAYOUTS))
def test_member_gemm_is_exact(probe, layout, tile_f, w2t):
    import torch
    rng = np.random.default_rng(10 + 2 * tile_f + w2t + 7 * LAYOUTS[layout])
    rows = ROWS[layout]
    # every feature column filled, the ones beyond K = 64 included (they must not be read); narrow: rows 32..63 are non-zero
    # and must not reach the 32 member rows of D
    A = _ints(rng, (rows, tile_f)) * _pow2(rng, rows)[:, None]
    W2 = _ints(rng, (H, H))
    W2 *= _pow2(rng, H)[None, :] if w2t else _pow2(rng, H)[:, None]      # one scale per B column: per j for A W2, per i for A W2'
    p = _weights()
    p[BLOCKS["W2"]] = W2.ravel(order="F")
    ref = A[:, :H] @ (W2 if w2t else W2.T)
    _assert_exact_in_fp32(ref)
    D = torch.full((MEMBERS[layout], H), float("nan"), dtype=torch.float32, device="cuda")
    pd, ad = _dev(p), _dev(A)                                          # held until the launch has finished
    _check(probe.probe_member_gemm(LAYOUTS[layout], tile_f, pd.data_ptr(), ad.data_ptr(), w2t, D.data_ptr()))
    got = _host(D)
    assert np.array_equal(got, ref[:got.shape[0]]), f"max |diff| {np.nanmax(np.abs(got - ref[:got.shape[0]]))}"


# ------------------------------------------------------------------------------------------------------------------------
# gradient GEMMs G1 += TA' TB, G2 += TH' TC and the store of their fragments into the parameter layout


def _grad_reference(TA, TB, TH, TC, K):
    """-> the 4482-entry gradient the fragments map to: G1 = sum_r TA_r' TB_r, G2 = sum_r TH_r' TC_r over the first K rows;
    rows 0..63 of G1 = wt dZ2 against [H1 | y0 y1 1]: dW2[i][j] = G1[i][j], db2[i] = G1[i][66]; rows 64..127 = wt dZ1:
    dW1[j][c] = G1[64 + j][64 + c], db1[j] = G1[64 + j][66]; G2 = [H2 | 1] against wt L: dW3[c][n] = G2[n][c], db3 = G2[64]."""
    G1 = np.einsum("rmf,rmg->fg", TA[:, :K], TB[:, :K])
    G2 = np.einsum("rmf,rmg->fg", TH[:, :K], TC[:, :K])
    return _pack(G1[64:, 64:66], G1[64:, 66], G1[:64, :64], G1[:64, 66], G2[:64, :2].T, G2[64, :2])


@pytest.mark.gpu
@pytest.mark.parametrize("R", [1, 3])
@pytest.mark.parametrize("layout", list(LAYOUTS))
def test_gradient_gemm_and_store_are_exact(probe, layout, R):
    """Every one of the 4482 entries is written (the buffer starts as NaN) and equals the exact contraction; R = 3 rounds
    with new tile contents accumulate in the register fragments.  Narrow: TA / TB rows 32..63 are non-zero and lie outside
    K = 32."""
    import torch
    rng = np.random.default_rng(100 + R + 10 * LAYOUTS[layout])
    rab, rhc, K = ROWS[layout], MEMBERS[layout], MEMBERS[layout]
    # one scale per feature column of each tile (fixed over the rounds): products of a (row, col) of G share one scale
    TA = _ints(rng, (R, rab, TA_F)) * _pow2(rng, TA_F)
    TB = _ints(rng, (R, rab, TB_F)) * _pow2(rng, TB_F)
    TH = _ints(rng, (R, rhc, TA_F)) * _pow2(rng, TA_F)
    TC = _ints(rng, (R, rhc, TC_F)) * _pow2(rng, TC_F)
    ref = _grad_reference(TA, TB, TH, TC, K)
    _assert_exact_in_fp32(ref)
    out = torch.full((P,), float("nan"), dtype=torch.float32, device="cuda")
    ts = [_dev(x) for x in (_weights(), TA, TB, TH, TC)]               # held until the launch has finished
    _check(probe.probe_grad_gemm(LAYOUTS[layout], ts[0].data_ptr(), R, *[t.data_ptr() for t in ts[1:]], out.data_ptr()))
    got = _host(out)
    assert not np.isnan(got).any(), f"entries never written: {np.flatnonzero(np.isnan(got))[:20]}"
    for name, sl in BLOCKS.items():
        assert np.array_equal(got[sl], ref[sl]), f"{name}: {np.flatnonzero(got[sl] != ref[sl])[:20]}"


# ------------------------------------------------------------------------------------------------------------------------
# one adjoint stage: tc_forward<true> + tc_backward<true> (tcw_ for the wide layout), then tc_grad_store


def _bf16(x):
    """round to nearest even bf16 (through fp32, as __floats2bfloat162_rn on an fp32 value)"""
    b = np.asarray(x, dtype=np.float32).view(np.uint32).astype(np.uint64)
    b = (b + 0x7FFF + ((b >> 16) & 1)) & 0xFFFF0000
    return b.astype(np.uint32).view(np.float32).astype(np.float64)


def _stage_reference(p, y, L, valid, wt, tanh=np.tanh):
    """fp64 emulation of one stage, rounded to bf16 exactly where the kernels round: H1 (tile TB), W2, wt dZ2 (TA), H2 (TH),
    wt dZ1 (TA), y (TB) and wt L (TC).  -> F[m][2], J[m][2], the CTA partial (wt-weighted gradient, 4482)."""
    W1, b1, W2, b2, W3, b3 = _unpack(p)
    W2b = _bf16(W2)
    H1 = _bf16(tanh(y @ W1.T + b1))
    h2 = tanh(H1 @ W2b.T + b2)
    F = h2 @ W3.T + b3
    wv = np.where(valid, wt, 0.0)[:, None]
    dZ2 = _bf16(wv * (L @ W3) * (1.0 - h2 * h2))
    dZ1 = (dZ2 @ W2b) * (1.0 - H1 * H1)
    J = (dZ1 @ W1) / wt
    dZ1b, H2b, yb, Lb = _bf16(dZ1), _bf16(h2), _bf16(y), _bf16(wv * L)
    partial = _pack(dZ1b.T @ yb, dZ1b.sum(0), dZ2.T @ H1, dZ2.sum(0), (H2b.T @ Lb).T, Lb.sum(0))
    return F, J, partial


def _stage_inputs(layout, seed):
    rng = np.random.default_rng(seed)
    M = MEMBERS[layout]
    y = rng.uniform(-2, 2, (M, 2)).astype(np.float32).astype(np.float64)
    L = rng.standard_normal((M, 2)).astype(np.float32).astype(np.float64)
    return y, L, np.ones(M, dtype=bool)


def _run_stage(probe, layout, p, y, L, valid, wt):
    import torch
    M = MEMBERS[layout]
    F = torch.full((M, 2), float("nan"), dtype=torch.float32, device="cuda")
    J = torch.full((M, 2), float("nan"), dtype=torch.float32, device="cuda")
    part = torch.full((P,), float("nan"), dtype=torch.float32, device="cuda")
    keep = [_dev(p), _dev(y), _dev(L), _dev(valid.astype(np.int32), torch.int32)]     # held until the launch has finished
    _check(probe.probe_stage(LAYOUTS[layout], *[t.data_ptr() for t in keep], float(wt), F.data_ptr(), J.data_ptr(), part.data_ptr()))
    return _host(F), _host(J), _host(part)


def _stage_bounds(p, y, L, valid, wt, trials=6, seed=7):
    """4x the largest deviation seen when every tanh of the emulation carries a random relative error of up to 2^-11
    (the documented bound of tanh.approx.f32), per output and per parameter block, plus 1e-5 of the block's largest
    magnitude for the fp32 (not fp64) sums of the kernels -- the only error of db3, which no tanh reaches."""
    rng = np.random.default_rng(seed)
    F0, J0, p0 = _stage_reference(p, y, L, valid, wt)
    spread = {"F": 0.0, "J": 0.0, **{k: 0.0 for k in BLOCKS}}
    for _ in range(trials):
        noisy = lambda x: np.tanh(x) * (1.0 + rng.uniform(-2.0 ** -11, 2.0 ** -11, np.shape(x)))
        F1, J1, p1 = _stage_reference(p, y, L, valid, wt, tanh=noisy)
        spread["F"] = max(spread["F"], np.abs(F1 - F0).max())
        spread["J"] = max(spread["J"], np.abs(J1 - J0).max())
        for k, sl in BLOCKS.items():
            spread[k] = max(spread[k], np.abs(p1[sl] - p0[sl]).max())
    ref = {"F": F0, "J": J0, **{k: p0[sl] for k, sl in BLOCKS.items()}}
    return {k: 4.0 * v + 1e-5 * np.abs(ref[k]).max() for k, v in spread.items()}, ref


# The derived bounds, relative to each output's largest magnitude (seed 1 weights, wt = 0.37):
#   narrow  F 1.1e-2  J 9.5e-3  W1 1.6e-2  b1 1.0e-2  W2 9.9e-3  b2 4.8e-3  W3 8.8e-3  b3 1e-5
#   wide    F 8.2e-3  J 1.4e-2  W1 1.6e-2  b1 1.1e-2  W2 1.5e-2  b2 7.4e-3  W3 1.5e-2  b3 1e-5
# They are NOT much tighter than the end-to-end 2e-2: a 2^-11 change of a tanh flips the bf16 rounding of about one H1 / H2
# entry in eight, and those one-ulp (2^-8) flips dominate.  The sharp checks of this path are the exact GEMM tests above
# and the exact relations below; this one catches errors of the size of a term (a lost 1/wt, a wrong tile half).
STAGE_REL_CEILING = 2e-2


@pytest.mark.gpu
@pytest.mark.parametrize("layout", list(LAYOUTS))
def test_one_stage_matches_the_bf16_emulation(probe, layout):
    p = _weights().astype(np.float32).astype(np.float64)
    y, L, valid = _stage_inputs(layout, 20 + LAYOUTS[layout])
    wt = 0.37                                          # a weight like h b_j: the VJP is divided by it again
    bounds, ref = _stage_bounds(p, y, L, valid, wt)
    F, J, part = _run_stage(probe, layout, p, y, L, valid, wt)
    got = {"F": F, "J": J, **{k: part[sl] for k, sl in BLOCKS.items()}}
    for k in ref:
        scale = np.abs(ref[k]).max()
        assert bounds[k] <= STAGE_REL_CEILING * scale, f"{k}: derived bound {bounds[k]:.3e} vs scale {scale:.3e}"
        err = np.abs(got[k] - ref[k]).max()
        assert err <= bounds[k], f"{k}: |device - emulation| {err:.3e} > derived bound {bounds[k]:.3e} (scale {scale:.3e})"


@pytest.mark.gpu
@pytest.mark.parametrize("layout", list(LAYOUTS))
def test_stage_weight_is_only_a_power_of_two_scale(probe, layout):
    """wt is folded into the cotangent side before every bf16 rounding and divided out of the VJP: for wt = 2^-k the VJP is
    bit-identical and the gradient partial is exactly 2^-k times the wt = 1 one."""
    p = _weights().astype(np.float32).astype(np.float64)
    y, L, valid = _stage_inputs(layout, 30 + LAYOUTS[layout])
    F1, J1, part1 = _run_stage(probe, layout, p, y, L, valid, 1.0)
    assert np.abs(part1).max() > 0
    for k in (0, 5, 20):
        F, J, part = _run_stage(probe, layout, p, y, L, valid, 2.0 ** -k)
        assert np.array_equal(F, F1), k
        assert np.array_equal(J, J1), k
        assert np.array_equal(part, part1 * 2.0 ** -k), k


@pytest.mark.gpu
@pytest.mark.parametrize("layout", list(LAYOUTS))
def test_stage_dead_members_contribute_nothing(probe, layout):
    """Members with valid = false (the pad rows of a ragged last CTA) holding large finite y and L leave the partial and the
    live members' F and J exactly as members holding zeros do."""
    p = _weights().astype(np.float32).astype(np.float64)
    y, L, valid = _stage_inputs(layout, 40 + LAYOUTS[layout])
    M = MEMBERS[layout]
    valid[::3] = False
    valid[-5:] = False
    dead = ~valid
    rng = np.random.default_rng(41)
    yb, Lb = y.copy(), L.copy()
    yb[dead] = rng.choice([-1.0, 1.0], (dead.sum(), 2)) * 1e3
    Lb[dead] = rng.choice([-1.0, 1.0], (dead.sum(), 2)) * 1e4
    yz, Lz = y.copy(), L.copy()
    yz[dead] = 0.0
    Lz[dead] = 0.0
    Fb, Jb, partb = _run_stage(probe, layout, p, yb, Lb, valid, 0.37)
    Fz, Jz, partz = _run_stage(probe, layout, p, yz, Lz, valid, 0.37)
    assert M - dead.sum() > 0 and np.isfinite(partb).all()
    assert (partb == partz).all()                      # value for value: +0 == -0
    assert (Jb[valid] == Jz[valid]).all() and (Fb[valid] == Fz[valid]).all()
