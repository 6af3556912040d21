"""A bf16-faithful twin of the tensor-core neural-ODE kernels (csrc/mlp_tc.cuh, 32 members per CTA; csrc/mlp_tc_wide.cuh,
128 members per CTA): the fixed-step Tsit5 forward pass and the InterpolatingAdjoint / GaussAdjoint reverse passes of the
C4 network f(u) = W3 tanh(W2 tanh(W1 u + b1) + b2) + b3, vectorised over the members, written from the numeric contract of
DESIGN section 4.5 and the Tsit5 tableau of tests/test_gpu_fixed_reference.Tab (not from the kernel loops).

Two modes:

* 'exact': np.longdouble, np.tanh, no rounding anywhere.  It restates mlp_restatement.restate('ld', ...) and so checks the
  twin's structure (stage sequence, dense outputs, Gauss nodes, cost jumps) independently of any kernel.
* 'bf16': the kernels' contract.
    - W1, b1, b2, W3, b3 are fp32; W2 is rounded to bf16.
    - first layer: fmaf(W1a, y0, fmaf(W1b, y1, b1)); H1 = bf16(tanh(.)).
    - Z2 = sum of bf16 products (exact in fp32), accumulated in fp32; H2 = tanh(fp32(Z2 + b2)) stays fp32;
      F = b3 + sum W3 H2 as fp32 fmaf chains in the layout's order (narrow: four 16-feature quarters from 0, then
      b3 + ((q0 + q1) + (q2 + q3)); wide: one 64-feature chain from b3).
    - stage inputs y and L, and lambda, are fp64 FMA combinations of fp32 values, rounded to fp32; the affine cotangent
      is a y + b in fp64, rounded to fp32, then added to lambda in fp32.
    - VJP: dZ2 = bf16(fp32(wt fmaf(W3a, L0, W3b L1)) (1 - H2^2)) with H2 in fp32; dZ1 = (dZ2 bf16(W2)) (1 - H1^2) with the
      bf16 H1; J = (W1' dZ1) (1 / wt), the sum in the layout's order.
    - gradient GEMMs: bf16(dZ2 | dZ1) against [H1 | bf16(y) | 1], bf16(H2) against bf16(wt L), fp32 registers per CTA over
      the whole reverse pass; mlp_reduce_kernel sums the fp32 CTA partials in fp64 and rounds to fp32.
    - InterpolatingAdjoint: wt = (float)(h b_s) at the six stages.  GaussAdjoint: seven stages without gradients (wt = 1),
      then the three nodes: lambda at hBq[g], y at hBq[2 - g], wt = (float)(h / 2 w_g).
  tanh is a callable on an fp32 array: the GPU tests pass the device's tanh.approx.f32, the CPU tests np.tanh rounded
  to fp32.

What the twin cannot reproduce is the accumulation order inside wgmma (Z2, dH1 and the gradient GEMMs).  It therefore
carries sum |terms| beside every such fp32 accumulation: the a-priori bound gamma_n sum |terms| for the gradient GEMMs,
and `perturb` (a numpy Generator) moves every member-GEMM result by a uniform random amount within the measured wgmma
residual (WGMMA_RESIDUAL x 2^-24 sum |terms|), so that the spread of the twin under perturbation measures what the
residual can do downstream (bf16 roundings it flips).

VARIANTS restate named wrong kernels for the separation guards.
"""
import os
import sys
from fractions import Fraction

import numpy as np

import mpmath as mp

HERE = os.path.dirname(os.path.abspath(__file__))
if HERE not in sys.path:
    sys.path.insert(0, HERE)

import mlp_restatement as R
import test_gpu_fixed_reference as FR
from ros23_restatement import C_TXT, b_exact

LD = np.longdouble
EPS32 = 2.0 ** -24
H = R.H
P = R.P
BLOCKS = R.BLOCKS
MEMBERS_PER_CTA = {"narrow": 32, "wide": 128}
TILES = ("H1", "dZ2", "dZ1", "H2", "y", "L")
VARIANTS = ("mirrored_gauss_nodes", "k6_for_k7", "lam_drops_ka6", "cost_component0", "no_start_ignored", "rz_H1", "rz_dZ2",
            "rz_all")
# the Gauss-Legendre node 1/2 (1 - sqrt(3/5)) as the restatement takes it
GAUSS_A = Fraction(1, 2) * (1 - Fraction(mp.nstr(mp.sqrt(mp.mpf("0.6")), 45)))
GAUSS_W = (Fraction(5, 9), Fraction(8, 9), Fraction(5, 9))


# The residual of the member GEMMs, calibrated from a measurement instead of the a-priori gamma_64 sum |terms|: on an H100
# the wgmma result of a 64-term bf16 product sum deviates from the exact sum by at most 4.9 x 2^-24 sum |terms| (mean 0.1
# for H1 W2', 0.5 for dZ2 W2; 22 % .. 69 % of the entries are the correctly rounded sum), over 20 GEMMs of realistic
# operands per layout and tile.  The twin perturbs by up to 8 x 2^-24 sum |terms| (the measured largest, rounded up to a
# power of two); tests/test_gpu_mlp_bf16_reference.py::test_member_gemm_residual_is_within_the_twins_model keeps the
# measurement within it.
WGMMA_RESIDUAL = 8.0


def gamma(n):
    """the a-priori relative bound of an n-term fp32 accumulation"""
    return n * EPS32 / (1.0 - n * EPS32)


def f32(x):
    """round to fp32 (returned as fp64 values)"""
    return np.asarray(x, dtype=np.float64).astype(np.float32).astype(np.float64)


def bf16(x, rz=False):
    """the fp32 values x rounded to bf16 as __floats2bfloat162_rn does (to nearest, ties to even; rz: toward zero, as
    __float2bfloat16_rz), returned as fp64 values"""
    b = np.asarray(x, dtype=np.float32).view(np.uint32).astype(np.uint64)
    if not rz:
        b = b + 0x7FFF + ((b >> 16) & 1)
    return (b & 0xFFFF0000).astype(np.uint32).view(np.float32).astype(np.float64)


def tanh_f32(x):
    """np.tanh of the fp32 arguments rounded to fp32: the CPU stand-in for tanh.approx.f32"""
    return f32(np.tanh(np.asarray(x, dtype=np.float64)))


def fmaf(a, b, c):
    """fp32 fmaf on fp32 values: a b is exact in fp64, the sum rounds once in fp64 and again to fp32 (a double rounding
    that differs from fmaf only when the fp64 sum lands exactly on an fp32 midpoint)"""
    return f32(a * b + c)


class Tables:
    """hA[7][6], hBst[4][7], hBq[3][7], hGW[3] of csrc/ode_tsit5.cuh: in long double from the exact tableau ('exact', h as
    the restatement takes it), or as the host builds them, fp64 products of h and the fp64 tableau ('bf16')"""

    def __init__(self, h, exact):
        kind = FR.Kind("ld")
        tab = FR.Tab(kind)
        if exact:
            hh = kind.const(h)
            conv = lambda fr: kind.const(fr)
        else:
            hh = np.float64(h)
            conv = lambda fr: np.float64(float(fr))
        self.hA = np.zeros((7, 6), dtype=LD if exact else np.float64)
        for s in range(7):
            for j, a in enumerate(tab.A[s] if exact else [Fraction(v) for v in FR.A_TXT[s]]):
                self.hA[s, j] = hh * (a if exact else np.float64(float(a)))
        thst = [1 - Fraction(C_TXT[s]) for s in range(1, 5)]
        thq = [GAUSS_A, Fraction(1, 2), 1 - GAUSS_A]
        self.hBst = np.array([[hh * conv(b_exact(j, t)) for j in range(7)] for t in thst])
        self.hBq = np.array([[hh * conv(b_exact(j, t)) for j in range(7)] for t in thq])
        self.hGW = np.array([hh / 2 * conv(w) for w in GAUSS_W])


class Twin:
    """one run of the twin over M members: p flat [P]; mode 'exact' or 'bf16'; layout 'narrow' / 'wide' (the order of
    the F and J sums, the chain length of the gradient GEMMs); perturb: None or a numpy Generator"""

    def __init__(self, p, h, mode="bf16", tanh=tanh_f32, layout="narrow", variant=None, perturb=None):
        assert mode in ("exact", "bf16") and layout in MEMBERS_PER_CTA and (variant is None or variant in VARIANTS)
        self.exact, self.layout, self.variant, self.rng = mode == "exact", layout, variant, perturb
        self.tanh = np.tanh if self.exact else tanh
        self.dt = LD if self.exact else np.float64
        self.tb = Tables(h, self.exact)
        p = np.asarray(p, dtype=np.float64)
        if not self.exact:
            p = f32(p)
        W1, b1, W2, b2, W3, b3 = (np.asarray(x, dtype=self.dt) for x in R.unpack(p))
        self.W1a, self.W1b, self.b1, self.b2, self.W3a, self.W3b, self.b3 = W1[:, 0], W1[:, 1], b1, b2, W3[0], W3[1], b3
        self.W2 = W2 if self.exact else bf16(W2)

    # ---- rounding points ----
    def r32(self, x):
        return x if self.exact else f32(x)

    def bf(self, x, tile):
        if self.exact:
            return x
        v = self.variant or ""
        return bf16(x, rz=v == "rz_all" or v == f"rz_{tile}")

    def fma(self, a, b, c):
        return a * b + c if self.exact else fmaf(a, b, c)

    def member_gemm(self, A, X):
        """A X with A [64][64] bf16, X [64][M] bf16: fp64 (exact), rounded to fp32; perturbed within WGMMA_RESIDUAL x 2^-24
        sum |terms| when the twin is perturbed"""
        Z = A @ X
        if self.exact:
            return Z
        if self.rng is not None:
            Z = Z + self.rng.uniform(-1.0, 1.0, Z.shape) * WGMMA_RESIDUAL * EPS32 * (np.abs(A) @ np.abs(X))
        return f32(Z)

    def chain(self, coef, vals, start):
        """sum_n coef[n] vals[n] over the 64 features as the layout sums it (fp32 fmaf chains); start = b3 (F) or 0 (J)"""
        if self.exact:
            return start + coef @ vals
        if self.layout == "wide":
            acc = np.broadcast_to(f32(start), vals.shape[1:]).astype(np.float64)
            for n in range(H):
                acc = fmaf(coef[n], vals[n], acc)
            return acc
        q = []
        for w in range(4):
            acc = np.zeros(vals.shape[1:])
            for n in range(16 * w, 16 * w + 16):
                acc = fmaf(coef[n], vals[n], acc)
            q.append(acc)
        return f32(start + f32(f32(q[0] + q[1]) + f32(q[2] + q[3])))

    # ---- the network ----
    def f(self, y):
        """F = f(y) for y [2][M]; -> (F [2][M], the point (y, H1, H2) for vjp)"""
        y = np.asarray(y, dtype=self.dt)
        z1 = self.fma(self.W1a[:, None], y[0][None], self.fma(self.W1b[:, None], y[1][None], self.b1[:, None]))
        H1 = self.bf(self.tanh(z1), "H1")
        H2 = self.tanh(self.r32(self.member_gemm(self.W2, H1) + self.b2[:, None]))
        F = np.array([self.chain(self.W3a, H2, self.b3[0]), self.chain(self.W3b, H2, self.b3[1])])
        return F, (y, H1, H2)

    def vjp(self, pt, L, wt, g=None, cnt=None):
        """J = (df/dy)' L at pt; with g (a dict of fp64 sums), adds the stage's wt-weighted parameter VJP and its sum of
        |terms|, each member weighed by cnt"""
        y, H1, H2 = pt
        L = np.asarray(L, dtype=self.dt)
        if self.exact:
            wt = self.dt(wt)
            dZ2 = wt * (self.W3a[:, None] * L[0] + self.W3b[:, None] * L[1]) * (1 - H2 * H2)
        else:
            wt = float(np.float32(wt))
            g3 = fmaf(self.W3a[:, None], L[0][None], f32(self.W3b[:, None] * L[1][None]))
            dZ2 = f32(f32(wt * g3) * f32(1.0 - H2 * H2))
        dZ2 = self.bf(dZ2, "dZ2")
        dZ1 = self.r32(self.member_gemm(self.W2.T, dZ2) * self.r32(1 - H1 * H1))
        inv = 1 / wt if self.exact else float(np.float32(1.0 / wt))
        J = np.array([self.r32(self.chain(self.W1a, dZ1, 0.0) * inv), self.r32(self.chain(self.W1b, dZ1, 0.0) * inv)])
        if g is not None:
            c = np.ones(y.shape[1]) if cnt is None else np.asarray(cnt, dtype=np.float64)
            if not self.exact:
                c = c.astype(np.float64)
            T1 = self.bf(dZ1, "dZ1")
            Y = self.bf(y, "y")
            Lw = self.bf(self.r32(wt * L), "L")
            H2b = self.bf(H2, "H2")
            one = np.ones((1, y.shape[1]), dtype=self.dt)
            # dW1[j][c], db1[j], dW2[i][j], db2[i], dW3[c][n], db3[c]: (cotangent-side tile) x (feature-side tile) over members
            pairs = {"W1": (T1, Y), "b1": (T1, one), "W2": (dZ2, H1), "b2": (dZ2, one), "W3": (Lw, H2b), "b3": (Lw, one)}
            for name, (A, B) in pairs.items():
                for key, f in (("g", lambda x: x), ("abs", np.abs)):
                    g[key][name] = g[key][name] + ((f(A) * c) @ f(B).T).reshape(g[key][name].shape)
        return J

    # ---- the passes ----
    def forward(self, u0, S):
        """-> (us [S+1][2][M], Ks [S][7][2][M]: k1..k6 and k7 = f(u_{n+1}))"""
        tb = self.tb
        u = np.asarray(u0, dtype=self.dt)
        u = self.r32(u)
        us, Ks = [u], []
        k0 = self.f(u)[0]
        for n in range(S):
            k = [k0]
            for sg in range(1, 7):
                y = self.r32(u + sum(tb.hA[sg, j] * k[j] for j in range(sg)))
                F = self.f(y)[0]
                k.append(F)
            us.append(y)
            Ks.append(k)
            u, k0 = y, k[6]
        return np.array(us), np.array(Ks)

    def stages(self, us):
        """the stages k1..k7 of every step of the trajectory us [S+1][2][M], one twin step from each us[n]"""
        S, M = us.shape[0] - 1, us.shape[2]
        Ks = self.forward(us[:-1].transpose(1, 0, 2).reshape(2, S * M), 1)[1][0]     # [7][2][S M]
        return Ks.reshape(7, 2, S, M).transpose(2, 0, 1, 3)

    def cotangent(self, lam, k, y, cost, dLdu):
        if isinstance(cost, str):
            d = np.asarray(dLdu[k], dtype=self.dt)
            return self.r32(lam + (d if self.exact else f32(d)))
        a, b = (np.broadcast_to(np.asarray(v, dtype=np.float64), (2,)) for v in cost)
        if self.variant == "cost_component0":
            a, b = np.array([a[0], a[0]]), np.array([b[0], b[0]])
        if self.exact:
            a, b = ([FR.Kind("ld").const(float(x)) for x in v] for v in (a, b))
        return self.r32(lam + self.r32(np.array([a[c] * y[c] + b[c] for c in range(2)])))

    def reverse(self, us, Ks, sos, cost, dLdu=None, sensealg="interpolating", no_start=False, cnt=None):
        """-> (du0 [2][M], dp [P], sum |terms| of dp [P], chain length of the gradient GEMMs in one CTA)"""
        tb = self.tb
        S = len(Ks)
        M = us.shape[2]
        zero = lambda shape: np.zeros(shape, dtype=self.dt)
        shapes = {"W1": (H, 2), "b1": (H,), "W2": (H, H), "b2": (H,), "W3": (2, H), "b3": (2,)}
        g = {key: {k: zero(s) for k, s in shapes.items()} for key in ("g", "abs")}
        gauss = sensealg == "gauss"
        lam = zero((2, M))
        if S in sos:
            lam = self.cotangent(lam, sos[S], us[S], cost, dLdu)
        for n in range(S - 1, -1, -1):
            uhi, ulo, kf = us[n + 1], us[n], list(Ks[n])
            kd = kf[:6] + [kf[5]] if self.variant == "k6_for_k7" else kf        # the reverse dense output's stages
            ka = []
            for sg in range(7 if gauss else 6):
                L = self.r32(lam + sum(tb.hA[sg, j] * ka[j] for j in range(min(sg, 6))))
                if sg == 0:
                    y = uhi
                elif sg >= 5:
                    y = ulo
                else:
                    y = self.r32(ulo + sum(tb.hBst[sg - 1, j] * kd[j] for j in range(7)))
                pt = self.f(y)[1]
                if gauss:
                    ka.append(self.vjp(pt, L, 1.0))
                else:
                    ka.append(self.vjp(pt, L, tb.hA[6, sg], g, cnt))
            if gauss:
                nl = 6 if self.variant == "lam_drops_ka6" else 7
                for gq in range(3):
                    gy = gq if self.variant == "mirrored_gauss_nodes" else 2 - gq
                    L = self.r32(lam + sum(tb.hBq[gq, j] * ka[j] for j in range(nl)))
                    y = self.r32(ulo + sum(tb.hBq[gy, j] * kd[j] for j in range(7)))
                    self.vjp(self.f(y)[1], L, tb.hGW[gq], g, cnt)
            lam = self.r32(lam + sum(tb.hA[6, j] * ka[j] for j in range(6)))
            if n in sos and not (no_start and n == 0 and self.variant != "no_start_ignored"):
                lam = self.cotangent(lam, sos[n], ulo, cost, dLdu)
        flat = lambda d: np.concatenate([d["W1"].ravel(order="F"), d["b1"], d["W2"].ravel(order="F"), d["b2"],
                                         d["W3"].ravel(order="F"), d["b3"]])
        dp, dabs = flat(g["g"]), flat(g["abs"])
        if not self.exact:
            dp = f32(dp)
        chain = S * (3 if gauss else 6) * MEMBERS_PER_CTA[self.layout] // 16
        return lam, dp, dabs, chain


def run(p, u0, h, S, sos, cost, dLdu=None, sensealg="interpolating", no_start=False, cnt=None, us=None, **kw):
    """forward over S steps from u0 [2][M], then the reverse pass with the save table sos {n: k}; -> dict(us, du0, dp,
    dp_abs, chain).  us [S+1][2][M] given (a kernel's own checkpoints): the reverse pass runs over them, its forward
    stages rebuilt by one twin step from each.  That approximates the stages the kernel's reverse pass reads back from its
    forward pass (a.kst): one twin step agrees with the kernel's next checkpoint to a few 1e-5, not bit for bit, and the
    perturbed twin rebuilds them too, so the spread covers the difference.
    kw: Twin's mode, tanh, layout, variant, perturb"""
    tw = Twin(p, h, **kw)
    if us is None:
        us, Ks = tw.forward(u0, S)
    else:
        us = np.asarray(us, dtype=tw.dt)
        Ks = tw.stages(us)
    du0, dp, dabs, chain = tw.reverse(us, Ks, sos, cost, dLdu, sensealg, no_start, cnt)
    f64 = lambda x: np.asarray(x, dtype=np.float64)
    return dict(us=f64(us), du0=f64(du0), dp=f64(dp), dp_abs=f64(dabs), chain=chain)


def dp_accumulation_bound(res):
    """the a-priori fp32 term of dp: the CTA's register chain of gradient MMAs (each adds a 16-member product), the fp32
    rounding of the CTA partial and of the reduced dp: gamma_{chain + 16 + 2} sum |terms|"""
    return gamma(res["chain"] + 18) * res["dp_abs"]


def spread(runner, base, trials=3, seed=0):
    """the largest deviation of the perturbed twin from base over `trials` runs of runner(perturb=rng): us and du0 in
    units of each member's largest |value| (pooled over members), dp per parameter block (absolute)"""
    rng = np.random.default_rng(seed)
    out = {"us": 0.0, "du0": 0.0, **{k: 0.0 for k in BLOCKS}}
    for _ in range(trials):
        r = runner(perturb=rng)
        for key in ("us", "du0"):
            if key in r and key in base:
                sc = member_scale(base[key])
                out[key] = max(out[key], float((np.abs(r[key] - base[key]) / sc).max()))
        if "dp" in r and "dp" in base:
            for k, sl in BLOCKS.items():
                out[k] = max(out[k], float(np.abs(r["dp"][sl] - base["dp"][sl]).max()))
    return out


def member_scale(x):
    """the largest |x| of each member over every other axis (members last), never 0"""
    x = np.abs(np.asarray(x, dtype=np.float64))
    sc = x.reshape(-1, x.shape[-1]).max(axis=0)
    return np.where(sc > 0, sc, 1e-300)


def derive(runner, trials=3, seed=0):
    """the twin's result and its derived bounds.  runner(perturb=...) -> a dict of run() (or a subset of its keys).
    Bounds: us / du0 in units of each member's largest |value|, 4x the perturbed spread; dp per parameter, the a-priori
    accumulation term plus 4x its block's perturbed spread"""
    base = runner(perturb=None)
    sp = spread(runner, base, trials, seed)
    bounds = {k: 4.0 * sp[k] for k in ("us", "du0")}
    if "dp" in base:
        b = dp_accumulation_bound(base)
        for k, sl in BLOCKS.items():
            b[sl] += 4.0 * sp[k]
        bounds["dp"] = b
    return base, bounds


CEILING = 1e-3          # every derived bound, relative to its output's scale


def ceilings(base, bounds):
    """each derived bound relative to its output's scale: us / du0 (already member-relative), dp per block (over the
    block's largest |dp|)"""
    out = {k: bounds[k] for k in ("us", "du0") if k in bounds}
    if "dp" in bounds:
        for k, sl in BLOCKS.items():
            out[k] = float(bounds["dp"][sl].max() / max(np.abs(base["dp"][sl]).max(), 1e-300))
    return out


def ratios(got, base, bounds, cols=None):
    """observed / bound per output: us / du0 per member and component (member m of got against twin member cols[m]),
    dp per parameter; -> {output: largest ratio}"""
    out = {}
    for k in ("us", "du0"):
        if k in got and k in bounds:
            ref = base[k] if cols is None else base[k][..., cols]
            err = np.abs(np.asarray(got[k], dtype=np.float64) - ref) / member_scale(ref)
            out[k] = float(err.max() / bounds[k]) if bounds[k] > 0 else (0.0 if err.max() == 0 else np.inf)
    if "dp" in got and "dp" in bounds:
        err = np.abs(np.asarray(got["dp"], dtype=np.float64) - base["dp"])
        for k, sl in BLOCKS.items():
            b = bounds["dp"][sl]
            out[k] = float(np.max(np.where(b > 0, err[sl] / np.where(b > 0, b, 1.0), np.where(err[sl] > 0, np.inf, 0.0))))
    return out
