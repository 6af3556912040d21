"""The SDE restatement of tests/sde_restatement.py checked on its own, and the CPU oracle checked against it (no GPU).

* Philox4x32-10 reproduces the published Random123 known-answer vectors (counter 0 / key 0, all ones, the pi digits).
* On the linear Stratonovich SDE du = p0 u dt + p1 u o dW (test/SDE1/sde_stratonovich.jl:22-113) the restated EulerHeun
  solution and its BacksolveAdjoint gradient approach the closed form u0 exp(p0 t + p1 W(t)) and
  dL/dp0 = sum_k t_k |u(t_k)|^2, dL/dp1 = sum_k W(t_k) . u(t_k)^2, dL/du0 = sum_k u(t_k)^2 / u0 (L = 1/2 sum_k |u(t_k)|^2)
  as dt shrinks, at strong order one: one Brownian path per member (Philox increments on the finest grid, summed to
  the coarser ones).
* oracle/adjoint_oracle.c against the 40-digit restatement over the configuration matrix of tests/sde_restatement.py
  (both families x EM / EulerHeun x Backsolve with each checkpoint mode and Interpolating with and without no_start x
  scalar affine, vector affine plus dgdp, explicit cost x shared and per-member p x four save-time sets, every pair of
  levels), 4 members, 40 steps of dt = 0.025, the same Philox increments on both sides: du0 and dp per member and
  component at 1e-12 relative, the component floored at 1e-6 of the member's largest.  Largest error observed: 1.8e-14
  (0.018 of the bound); the module takes about 12 s of host time.
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
from oracle import oracle as O

# Random123 kat_vectors, philox4x32 10: counter words, key words, output words
KAT = [((0x00000000, 0x00000000, 0x00000000, 0x00000000), (0x00000000, 0x00000000), (0x6627e8d5, 0xe169c58d, 0xbc57ac4c, 0x9b00dbd8)),
       ((0xffffffff, 0xffffffff, 0xffffffff, 0xffffffff), (0xffffffff, 0xffffffff), (0x408f276d, 0x41c83b0e, 0xa20bc7c6, 0x6d5451fd)),
       ((0x243f6a88, 0x85a308d3, 0x13198a2e, 0x03707344), (0xa4093822, 0x299f31d0), (0xd16cfe09, 0x94fdcceb, 0x5001e420, 0x24126ea1))]


@pytest.mark.parametrize("ctr,key,out", KAT)
def test_philox_known_answers(ctr, key, out):
    assert tuple(int(w) for w in R.philox4x32_10(ctr, key)) == out


def test_uniforms_round_like_float64_above_two_to_the_52():
    """a >= 2^52: (double)a + 0.5 is a tie and rounds to even, so an odd a lands on a + 1 and the largest word,
    a = 2^53 - 1, on exactly 1.0; the smallest uniform is 2^-54.  So the uniforms lie in (0, 1], and u1 = 1 gives
    rad = sqrt(-2 log 1) = 0, a finite normal pair (0, 0), never a NaN."""
    r = [np.array([0xFFFFFFFF, 0x80000000, 0x80000000, 0]), np.array([0xFFFFFFFF, 0x00000800, 0x00001000, 0]),
         np.array([0, 0, 0, 0]), np.array([0, 0, 0, 0])]
    u1, u2 = R.uniforms([np.asarray(x, dtype=np.uint64) for x in r])
    a = [(2 ** 53 - 1), (1 << 52) + 1, (1 << 52) + 2, 0]
    expect = [float(x) + 0.5 for x in a]                 # Python floats round the same way (IEEE round-to-nearest-even)
    assert list(u1) == [e * 2.0 ** -53 for e in expect]
    assert u1[0] == 1.0 and u1[1] == u1[2] == (2 ** 52 + 2) * 2.0 ** -53 and u1[3] == 2.0 ** -54 and (u2 == 2.0 ** -54).all()
    z0, z1, rad = R.box_muller(u1, u2, "mp")
    assert rad[0] == 0 and z0[0] == 0 and z1[0] == 0 and all(np.isfinite(float(v)) for v in list(z0) + list(z1))


def test_linear_stratonovich_converges_to_the_closed_form():
    M, T, fine = 16, 1.0, 512
    p = np.array([1.01, 0.87])
    u0 = np.array([[1.0], [0.5]]) * np.ones((2, M))
    dWf, _ = R.increments(1, 0, M, fine, 2, T / fine, "ld")
    dWf = dWf.astype(np.float64)
    errs = []
    for S in (32, 64, 128, 256):
        r = fine // S
        dW = dWf.reshape(S, r, 2, M).sum(1)
        h = T / S
        saveat = np.linspace(0.0, T, S + 1)[:: S // 8]
        du0, dp, us = R.gradient("ld", "sde_linear", "euler_heun", "backsolve", u0, p, dW, h, saveat, cost=("affine", 1.0, 0.0))
        W = np.concatenate([np.zeros((1, 2, M)), np.cumsum(dW, 0)], 0)
        idx = np.round(saveat / h).astype(int)
        ex = u0[None] * np.exp(p[0] * saveat[:, None, None] + p[1] * W[idx])
        gp0 = (saveat[:, None, None] * ex ** 2).sum((0, 1))
        gp1 = (W[idx] * ex ** 2).sum((0, 1))
        gu0 = (ex ** 2 / u0[None]).sum(0)
        e = [np.abs(us[idx] - ex).max() / np.abs(ex).max(), np.abs(dp.sum(1) - [gp0.sum(), gp1.sum()]).max() / np.abs(gp0.sum()),
             np.abs(du0 - gu0).max() / np.abs(gu0).max()]
        errs.append(e)
    errs = np.array(errs)
    print("relative errors (state, dp, du0) at S = 32 .. 256:\n", errs)
    assert (errs[1:] / errs[:-1] < 0.7).all(), errs          # strong order one: halving dt roughly halves every error
    assert errs[-1].max() < 1e-2


@pytest.mark.parametrize("c", R.config_matrix(), ids=R.label)
def test_oracle_matches_the_40_digit_restatement(c):
    N = 4
    u0, p, cost, dgdp, dLdu = R.problem(c, N, seed=11)
    sensealg, ckpt, no_start = R.SENSEALGS[c["sa"]]
    saveat = R.SAVEATS[c["saveat"]]
    dW, _ = R.increments(77, 5, N, R.S_STEPS, 2, R.H, "ld")
    dW = dW.astype(np.float64)
    du0, dp, _ = R.gradient("mp", c["family"], c["stepper"], sensealg, u0, p, dW, R.H, saveat, cost=cost, dLdu=dLdu,
                            dgdp=dgdp, ckpt=ckpt, no_start=no_start)
    kw = dict(cost=("explicit",) if cost[0] == "explicit" else ("affine", 0.0, 0.0), shared_p=c["p"] == "shared",
              no_start=no_start, checkpointing=ckpt != "never", ckpt_every_step=ckpt == "every", d=2)
    if cost[0] == "affine":
        kw["cost_vec"] = (cost[1], cost[2]) + (() if dgdp is None else dgdp)
    cfg = O.make_cfg(c["family"], sensealg, c["stepper"], N, saveat, 0.0, R.T_END, dt=R.H, **kw)
    ref = O.gradient(cfg, saveat, u0, p, dLdu=dLdu, dW=dW)
    dp_ref = dp.sum(1) if c["p"] == "shared" else dp
    e = max(R.rel_err(ref["du0"], du0).max(), R.rel_err(ref["dp"], dp_ref).max())
    print(f"{R.label(c)}: oracle vs 40 digits {e:.2e}")
    assert e < 1e-12
