"""The CUDA-core neural-ODE device functions (csrc/mlp.cuh: mlp_load_params, mlp_gemm, mlp_forward, mlp_backward,
mlp_accumulate, mlp_store_grad, mlp_reduce_kernel), one block at a time, through tests/csrc/mlp_probe.cu, for
T = double and T = float.

* Exact, bit for bit: mlp_gemm on small integers (both weight images, W2 and W2'); mlp_accumulate + mlp_store_grad on
  integer activations and a power-of-two weight c, so the gradient is an exact integer sum placed at its column-major
  slot (every one of the 4482 store positions), for nvalid in {1, 17, 31, 32} with large distinct values in the pad
  columns, which would show in the sums if they leaked; mlp_reduce_kernel: the block partials summed in block order in
  fp64, i.e. the sequential fp64 sum (double) and float(the sequential double sum) (float).
* With tanh: mlp_forward (H1, H2, F) against the long-double network of tests/mlp_restatement.py, and mlp_backward
  (D2, D1, J' L) against long double on the device's own activations.  The bounds are propagated from CUDA's documented
  accuracy of tanh / tanhf (2 ulp, CUDA Math API, Appendix "Mathematical Functions") and the unit roundoff u of every
  fma chain (gamma_n = n u / (1 - n u)), element by element; a factor 2 covers the second-order terms.
"""
import ctypes as C
import os
import subprocess
import sys

import numpy as np
import pytest

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(HERE)
for d in (ROOT, HERE):
    if d not in sys.path:
        sys.path.insert(0, d)

from scimlsensitivity_jl_b200 import _lib

import mlp_restatement as R

CSRC = os.path.join(ROOT, "scimlsensitivity.jl_b200", "csrc")
PROBE = os.path.join(ROOT, "tests", "csrc", "mlp_probe.cu")
H, TB, P = 64, 32, R.P
DTYPES = {"f64": np.float64, "f32": np.float32}
UNIT = {"f64": 2.0 ** -53, "f32": 2.0 ** -24}
NAMES = ("probe_gemm", "probe_layers", "probe_accumulate", "probe_reduce")


@pytest.fixture(scope="session")
def probe_so(tmp_path_factory):
    """mlp_probe.cu built with the library's own nvcc flags, once per session, outside the source tree."""
    so = str(tmp_path_factory.mktemp("mlp_probe") / "libmlp_probe.so")
    cmd = [_lib.nvcc_path(), "-gencode", "arch=compute_90a,code=sm_90a", "-O3", "-std=c++17", "-I", CSRC,
           "-Xcompiler", "-fPIC", "-shared", PROBE, "-o", so]
    res = subprocess.run(cmd, capture_output=True, text=True)
    assert res.returncode == 0, res.stdout[-3000:] + res.stderr[-3000:]
    return so


def test_probe_compiles_for_sm90a(probe_so):
    """No GPU needed: a header change that breaks the probes fails here."""
    assert os.path.getsize(probe_so) > 0
    lib = C.CDLL(probe_so)
    for name in NAMES:
        for sfx in ("f64", "f32"):
            getattr(lib, f"{name}_{sfx}")


@pytest.fixture(scope="module")
def probe(probe_so):
    lib = C.CDLL(probe_so)
    vp = C.c_void_p
    for sfx, ct in (("f64", C.c_double), ("f32", C.c_float)):
        getattr(lib, f"probe_gemm_{sfx}").argtypes = [vp, vp, C.c_int, vp]
        getattr(lib, f"probe_layers_{sfx}").argtypes = [vp] * 9
        getattr(lib, f"probe_accumulate_{sfx}").argtypes = [vp] * 6 + [ct, C.c_int, vp]
        getattr(lib, f"probe_reduce_{sfx}").argtypes = [vp, vp, C.c_int]
        for n in NAMES:
            getattr(lib, f"{n}_{sfx}").restype = C.c_int
    return lib


def _dev(x, dtype):
    import torch
    return torch.tensor(np.ascontiguousarray(x, dtype=DTYPES[dtype]), device="cuda")


def _empty(shape, dtype):
    import torch
    return torch.full(shape, float("nan"), dtype=torch.float64 if dtype == "f64" else torch.float32, device="cuda")


def _host(t):
    return t.cpu().numpy().astype(np.float64)


def _check(rc):
    assert rc == 0, f"probe launch failed: cudaError {rc}"


def _ints(rng, shape, lo=-8, hi=8):
    return rng.integers(lo, hi + 1, size=shape).astype(np.float64)


def _gamma(n, u):
    return n * u / (1 - n * u)


@pytest.mark.gpu
@pytest.mark.parametrize("transposed", [0, 1], ids=["W2", "W2T"])
@pytest.mark.parametrize("dtype", list(DTYPES))
def test_gemm_is_exact(probe, dtype, transposed):
    rng = np.random.default_rng(3 + transposed + 2 * (dtype == "f32"))
    p = _ints(rng, P)
    X = _ints(rng, (H, TB))
    W2 = R.unpack(p)[2]                                       # W2[i][j]
    out = _empty((H, TB), dtype)
    dp_, dX = _dev(p, dtype), _dev(X, dtype)                 # held: a freed input's memory would be handed to the next one
    _check(getattr(probe, f"probe_gemm_{dtype}")(dp_.data_ptr(), dX.data_ptr(), transposed, out.data_ptr()))
    expect = (W2.T if transposed else W2) @ X
    assert np.array_equal(_host(out), expect)


@pytest.mark.gpu
@pytest.mark.parametrize("nvalid", [1, 17, 31, 32])
@pytest.mark.parametrize("dtype", list(DTYPES))
def test_accumulate_and_store_are_exact(probe, dtype, nvalid):
    rng = np.random.default_rng(100 + nvalid)
    c = 0.125
    y, L = _ints(rng, (2, TB)), _ints(rng, (2, TB))
    H1, H2, D1, D2 = (_ints(rng, (H, TB)) for _ in range(4))
    for k, a in enumerate((y, L, H1, H2, D1, D2)):            # pad columns: large and distinct, visible in any sum
        a[:, nvalid:] = 1024 + 64 * k + np.arange(nvalid, TB)
    out = _empty((P,), dtype)
    args = [_dev(a, dtype) for a in (y, L, H1, H2, D1, D2)]
    _check(getattr(probe, f"probe_accumulate_{dtype}")(*[a.data_ptr() for a in args], c, nvalid, out.data_ptr()))
    v = slice(0, nvalid)
    dW1 = c * D1[:, v] @ y[:, v].T                            # [i][c]
    db1, db2 = c * D1[:, v].sum(1), c * D2[:, v].sum(1)
    dW2 = c * D2[:, v] @ H1[:, v].T                           # [i][j]
    dW3 = c * L[:, v] @ H2[:, v].T                            # [c][j]
    db3 = c * L[:, v].sum(1)
    expect = np.concatenate([dW1.ravel(order="F"), db1, dW2.ravel(order="F"), db2, dW3.ravel(order="F"), db3])
    got = _host(out)
    bad = np.flatnonzero(got != expect)
    assert bad.size == 0, [(int(q), next(k for k, s in R.BLOCKS.items() if s.start <= q < s.stop), got[q], expect[q]) for q in bad[:8]]


@pytest.mark.gpu
@pytest.mark.parametrize("dtype", list(DTYPES))
def test_reduce_sums_blocks_in_order_in_fp64(probe, dtype):
    rng = np.random.default_rng(7)
    nb = 9
    parts = (rng.standard_normal((nb, P)) * np.exp2(rng.integers(-30, 30, (nb, P)))).astype(DTYPES[dtype]).astype(np.float64)
    out, dparts = _empty((P,), dtype), _dev(parts, dtype)
    _check(getattr(probe, f"probe_reduce_{dtype}")(dparts.data_ptr(), out.data_ptr(), nb))
    acc = np.zeros(P)
    for k in range(nb):
        acc = acc + parts[k]
    expect = acc if dtype == "f64" else acc.astype(np.float32).astype(np.float64)
    assert np.array_equal(_host(out), expect)
    # the order matters at these magnitudes: a pairwise or reversed sum differs somewhere
    rev = np.zeros(P)
    for k in reversed(range(nb)):
        rev = rev + parts[k]
    assert (rev != acc).any()


@pytest.mark.gpu
@pytest.mark.parametrize("dtype", list(DTYPES))
def test_forward_and_backward_against_long_double(probe, dtype):
    rng = np.random.default_rng(11 + (dtype == "f32"))
    cast = lambda x: np.asarray(x, dtype=DTYPES[dtype]).astype(np.float64)
    u = UNIT[dtype]
    p = cast(R.weights())
    y, L = cast(rng.uniform(-2, 2, (2, TB))), cast(rng.standard_normal((2, TB)))
    outs = {k: _empty(shape, dtype) for k, shape in (("F", (2, TB)), ("H1", (H, TB)), ("H2", (H, TB)), ("D2", (H, TB)),
                                                     ("D1", (H, TB)), ("JTL", (2, TB)))}
    ins = [_dev(a, dtype) for a in (p, y, L)]
    _check(getattr(probe, f"probe_layers_{dtype}")(*[a.data_ptr() for a in ins], *[outs[k].data_ptr() for k in ("F", "H1", "H2", "D2", "D1", "JTL")]))
    got = {k: _host(v) for k, v in outs.items()}
    W1, b1, W2, b2, W3, b3 = (np.asarray(a, dtype=np.float64) for a in R.unpack(p))
    LD = np.longdouble
    _, rH1, rH2, rF = R.layers([y[0].astype(LD), y[1].astype(LD)], p.reshape(-1, 1).astype(LD))
    rH1, rH2, rF = (np.asarray(a, dtype=np.float64) for a in (rH1, rH2, rF))
    tanh_err = lambda h: 2 * 2 * u * np.abs(h)               # 2 ulp, ulp(h) <= 2 u |h|
    aW1, aW2, aW3 = np.abs(W1), np.abs(W2), np.abs(W3)
    # forward: z1 = fma(W1_0, y0, fma(W1_1, y1, b1)); z2 = 64-fma chain + b2; F = b3 + 64-fma chain
    e1 = (1 - rH1 ** 2) * _gamma(2, u) * (aW1 @ np.abs(y) + np.abs(b1)[:, None]) + tanh_err(rH1)
    e2 = (1 - rH2 ** 2) * (aW2 @ e1 + _gamma(65, u) * (aW2 @ np.abs(rH1) + np.abs(b2)[:, None])) + tanh_err(rH2)
    eF = aW3 @ e2 + _gamma(65, u) * (aW3 @ np.abs(rH2) + np.abs(b3)[:, None])
    # backward on the device's own activations
    H1d, H2d, D2d, D1d = got["H1"], got["H2"], got["D2"], got["D1"]
    rD2 = np.asarray((W3.T.astype(LD) @ L.astype(LD)) * (1 - H2d.astype(LD) ** 2), dtype=np.float64)
    eD2 = _gamma(5, u) * (aW3.T @ np.abs(L)) * (1 + H2d ** 2)
    rD1 = np.asarray((W2.T.astype(LD) @ D2d.astype(LD)) * (1 - H1d.astype(LD) ** 2), dtype=np.float64)
    eD1 = _gamma(67, u) * (aW2.T @ np.abs(D2d)) * (1 + H1d ** 2)
    rJ = np.asarray(W1.T.astype(LD) @ D1d.astype(LD), dtype=np.float64)
    eJ = _gamma(64, u) * (aW1.T @ np.abs(D1d))
    worst = {}
    for k, ref, bound in (("H1", rH1, e1), ("H2", rH2, e2), ("F", rF, eF), ("D2", rD2, eD2), ("D1", rD1, eD1), ("JTL", rJ, eJ)):
        ratio = np.abs(got[k] - ref) / (2 * bound + 1e-300)
        worst[k] = float(ratio.max())
    print(f"{dtype}: largest error as a share of its bound", {k: float('%.2g' % v) for k, v in worst.items()})
    assert max(worst.values()) <= 1.0, worst
