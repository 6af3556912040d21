"""The neural-ODE family  f(u) = W3 tanh(W2 tanh(W1 u + b1) + b2) + b3  (2 -> 64 -> 64 -> 2, BASELINE config C4) restated
for the fixed-grid Tsit5 restatement of tests/test_gpu_fixed_reference.py, in 40-digit mpmath ('mp', object arrays) or
np.longdouble ('ld', vectorised over the members).

* The network in matrix form.  The parameters are the flat column-major layout [W1 | b1 | W2 | b2 | W3 | b3],
  P = 4482, shared by every member: the problem's p is one column [P][1].
* (df/dp)' lam by hand-written backprop from the formula (never from the kernels or the oracle): the reverse pass of
  the three layers, the weight blocks as outer products, stored at their column-major positions.  It is the family's
  vjp_p hook, so the restatement's mu stays one [P][M] array.  (df/du)' lam stays the restatement's complex step.
* restate(): the forward and reverse of test_gpu_fixed_reference.py with this family, plus the variants the separation
  guards compare against (mirrored Gauss nodes of the forward dense output, a linear dense output, event scales
  dropped in the reverse pass).
"""
import os
import sys
from fractions import Fraction

import numpy as np

import mpmath as mp

HERE = os.path.dirname(os.path.abspath(__file__))
if HERE not in sys.path:
    sys.path.insert(0, HERE)

import test_gpu_fixed_reference as FR

H, D = 64, 2
P = H * D + H + H * H + H + D * H + D                      # 4482
OW1, OB1 = 0, H * D
OW2 = OB1 + H
OB2 = OW2 + H * H
OW3 = OB2 + H
OB3 = OW3 + D * H
BLOCKS = {"W1": slice(OW1, OB1), "b1": slice(OB1, OW2), "W2": slice(OW2, OB2), "b2": slice(OB2, OW3), "W3": slice(OW3, OB3),
          "b3": slice(OB3, P)}


def weights(seed=1):
    """the C4 network of tests/test_gpu_parity_mlp.py (_weights), flat column-major"""
    rng = np.random.default_rng(seed)
    W1 = rng.standard_normal((H, 2)) / np.sqrt(2); W2 = rng.standard_normal((H, H)) / np.sqrt(H); W3 = rng.standard_normal((2, H)) / np.sqrt(H)
    b1, b2, b3 = 0.1 * rng.standard_normal(H), 0.1 * rng.standard_normal(H), 0.1 * rng.standard_normal(2)
    return np.concatenate([W1.ravel(order="F"), b1, W2.ravel(order="F"), b2, W3.ravel(order="F"), b3])


def unpack(q):
    """flat p (one member's column) -> W1[i][c], b1[i], W2[i][j], b2[i], W3[c][j], b3[c]"""
    return (q[OW1:OB1].reshape(D, H).T, q[OB1:OW2], q[OW2:OB2].reshape(H, H).T, q[OB2:OW3], q[OW3:OB3].reshape(H, D).T, q[OB3:P])


def _tanh(x):
    return np.vectorize(mp.tanh, otypes=[object])(x) if x.dtype == object else np.tanh(x)


def _col(b):
    return b.reshape(-1, 1)


def layers(y, p):
    """-> (U[2][M], H1[64][M], H2[64][M], F[2][M]) at the states y (list of D member arrays, real or complex)"""
    W1, b1, W2, b2, W3, b3 = unpack(np.asarray(p)[:, 0])
    U = np.array(list(y))
    H1 = _tanh(W1 @ U + _col(b1))
    H2 = _tanh(W2 @ H1 + _col(b2))
    return U, H1, H2, W3 @ H2 + _col(b3)


def backprop(y, p, lam):
    """the reverse pass of the three layers for the cotangent lam -> (D2, D1, J' lam, the [P][M] parameter VJP)"""
    W1, b1, W2, b2, W3, b3 = unpack(np.asarray(p)[:, 0])
    U, H1, H2, _ = layers(y, p)
    L = np.array(list(lam))
    D2 = (W3.T @ L) * (1 - H2 * H2)                    # d/dz2
    D1 = (W2.T @ D2) * (1 - H1 * H1)                   # d/dz1
    M = U.shape[1]
    # column-major blocks: W[i][j] at offset + j * rows + i, i.e. the [j][i] array flattened
    g = np.concatenate([(U[None, :, :] * D1[:, None, :]).transpose(1, 0, 2).reshape(D * H, M), D1,
                        (D2[:, None, :] * H1[None, :, :]).transpose(1, 0, 2).reshape(H * H, M), D2,
                        (L[:, None, :] * H2[None, :, :]).transpose(1, 0, 2).reshape(D * H, M), L])
    return D2, D1, W1.T @ D1, g


class MlpFamily:
    """f(y, p) for the restatement, with (df/dp)' lam as the vjp_p hook"""

    def __call__(self, y, p):
        return list(layers(y, p)[3])

    def vjp_p(self, kind, y, p, lam):
        return backprop(y, p, lam)[3]


MLP = MlpFamily()
FAMILY = (MLP, D, P)


def problem(h, S, u0, p, sos, cost, dLdu=None, events=None, no_start=False):
    """a restatement problem of the MLP family; u0[2][M], p flat [P] (shared), events {n: (s[2], c[2])}"""
    ev = {n: (s, c, None, None) for n, (s, c) in (events or {}).items()}
    return FR.Problem(FAMILY, h, S, np.asarray(u0, dtype=np.float64), np.asarray(p, dtype=np.float64).reshape(P, 1), sos, cost,
                      dLdu, ev, None, no_start)


class LinearTab(FR.Tab):
    """a linear dense output u_n + theta (u_{n+1} - u_n) in place of b_j(theta) (restates a wrong kernel)"""

    def b(self, th):
        return [self.kind.const(Fraction(th)) * w for w in super().b(1)]


VARIANTS = ("mirrored_gauss_nodes", "linear_dense", "no_event_scale")


def restate(kind_name, pr, sensealg, variant=None):
    """-> dict(us = checkpoints [S+1][2][M] (post-event), du0 [2][M], mu [P][M]); variant in VARIANTS restates a wrong
    kernel: the forward dense output at the mirrored Gauss node (theta in place of 1 - theta), a linear dense output,
    or lam- = lam+ at an event"""
    kind = FR.Kind(kind_name)
    ctx = mp.workdps(FR.DPS) if kind_name == "mp" else FR._nullctx()
    with ctx:
        tab = (LinearTab if variant == "linear_dense" else FR.Tab)(kind)
        us, Ks, ps = FR.forward(kind, tab, pr)
        rpr = pr
        if variant == "no_event_scale":
            rpr = FR.Problem(FAMILY, pr.h, pr.S, pr.u0, pr.p, pr.sos, pr.cost, pr.dLdu,
                             {n: (np.ones(D), c, a, b) for n, (s, c, a, b) in pr.events.items()}, None, pr.no_start)
        gy = (lambda tha: Fraction(tha)) if variant == "mirrored_gauss_nodes" else None
        lam, mu = FR.reverse(kind, tab, rpr, sensealg, us, Ks, ps, gauss_y=gy)
        return dict(us=np.array([[kind.f64(v) for v in u] for u in us]), du0=np.array([kind.f64(v) for v in lam]),
                    mu=np.array([kind.f64(v) for v in mu]))


def rel_err(got, ref, floor=1e-6):
    """per member and component: |got - ref| / max(|ref|, floor * the member's largest |ref|); arrays [C][M]"""
    return FR.rel_err(got, ref, floor)


# dp's floor: an fp64 sum of a block's terms rounds at about 1e-15 of the block's largest entry (the oracle: 3e-16 ..
# 9e-16 over the configuration matrix), so a floor of 1e-6 would ask 1e-18 of the block's scale at its smallest entries,
# below fp64.  1e-3 of the block's largest asks 1e-15 there and 1e-12 relative of every larger entry.
DP_FLOOR = 1e-3


def dp_err(got, ref, floor=DP_FLOOR):
    """per parameter, |got - ref| over max(|ref|, floor * the largest |ref| of its block) (the Rosenbrock23 reference's
    convention, block by block: a small block is not hidden under W2's scale); -> (largest, {block: largest})"""
    got, ref = np.asarray(got, dtype=np.float64).reshape(-1), np.asarray(ref, dtype=np.float64).reshape(-1)
    per = {}
    for name, sl in BLOCKS.items():
        r = ref[sl]
        scale = np.maximum(np.abs(r), floor * np.abs(r).max())
        scale = np.where(scale > 0, scale, 1e-300)
        per[name] = float(np.max(np.abs(got[sl] - r) / scale))
    return max(per.values()), per
