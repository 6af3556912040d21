"""General-noise SDE family plug-ins without a GPU (nvcc cross-compiles, a plug-in registers without touching the device).

* Each example plug-in of examples/sde_noise_families.cuh registers, and b200adj_family_noise, b200adj_family_noise_kind
  and FAMILIES report its (d, P, m) and general noise; the built-in and diagonal plug-in families report theirs.
* A family outside the limits (D or M outside 1..4, P outside 1..8) or without g_apply does not compile.
* The registry refuses a diagonal-noise plug-in with m != d, a general one with m > 4, an SDE plug-in without a noise kind
  and an ODE plug-in with one, whatever the headers let through.
* On the host, before any handle exists: a noise_rate_prototype of the wrong shape, or on a diagonal family, raises
  ValueError; EM + BacksolveAdjoint on a general family raises NotImplementedError; noisemixing = true is accepted for a
  general family and still refused for a diagonal plug-in.
"""
import os
import subprocess
import sys

import numpy as np
import pytest

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(HERE)
if ROOT not in sys.path:
    sys.path.insert(0, ROOT)

import scimlsensitivity_jl_b200 as b
from scimlsensitivity_jl_b200 import _lib
from scimlsensitivity_jl_b200.concrete_solve import _check_noise_rate_prototype
from scimlsensitivity_jl_b200.problems import FAMILY_CONDITIONS, GENERAL_NOISE_FAMILIES
from scimlsensitivity_jl_b200.sensitivity_interface import _check_general_noise, _check_noise_mixing

EXAMPLES = os.path.join(ROOT, "examples")
# examples/sde_noise_families.cuh: (name, d, P, m)
NOISE_FAMILIES = (("sde_roessler", 2, 4, 2), ("sde_mixing", 2, 4, 2), ("sde_additive", 2, 2, 2), ("sde_nonsquare", 3, 2, 2),
                  ("sde_scalar", 2, 2, 1), ("sde_lv_general", 2, 6, 2))


def _register(name):
    so = os.path.join(EXAMPLES, f"libb200fam_{name}.so")
    if not os.path.exists(so):
        pytest.skip("the example plug-ins are built by __graft_entry__.build()")
    return b.register_family(so)


@pytest.mark.parametrize("name,d,P,m", NOISE_FAMILIES, ids=[f[0] for f in NOISE_FAMILIES])
def test_example_plugin_registers_with_its_noise(name, d, P, m):
    fid, d_, P_ = _register(name)
    assert (d_, P_) == (d, P) and fid >= 100
    assert _lib.family_noise(fid) == m and _lib.family_noise_kind(fid) == _lib.NOISE_GENERAL
    assert b.FAMILIES[name] == (d, P, m) and FAMILY_CONDITIONS[name] == 0 and name in GENERAL_NOISE_FAMILIES


def test_noise_kind_of_the_other_families():
    kinds = {"lv": _lib.NOISE_NONE, "lorenz": _lib.NOISE_NONE, "robertson": _lib.NOISE_NONE, "sde_lv": _lib.NOISE_DIAGONAL,
             "mlp": _lib.NOISE_NONE, "sde_linear": _lib.NOISE_DIAGONAL, "ball": _lib.NOISE_NONE, "relax": _lib.NOISE_NONE}
    for name, k in kinds.items():
        assert _lib.family_noise_kind(_lib.FAM[name]) == k
    for bad in (8, 99, 100 + 10_000, -1):
        with pytest.raises(_lib.B200AdjError) as e:
            _lib.family_noise_kind(bad)
        assert e.value.code == -1
    fid, _, _ = _register("sde_chain3")
    assert _lib.family_noise_kind(fid) == _lib.NOISE_DIAGONAL and "sde_chain3" not in GENERAL_NOISE_FAMILIES


def _family(D, P, M, g_apply=True):
    """a general-noise struct: f = -u, G[i][j] = p0 u_i"""
    ga = ("    template <class T> __device__ __forceinline__ static void g_apply(const T* u, const T* p, const T* w, T* out) {\n"
          "        for (int i = 0; i < D; i++) { out[i] = 0; for (int j = 0; j < M; j++) out[i] += p[0] * u[i] * w[j]; } }\n") if g_apply else ""
    return (f"struct Probe {{\n    static constexpr int D = {D}, P = {P}, M = {M};\n"
            "    template <class T> __device__ __forceinline__ static void f(const T* u, const T* p, T* du) { for (int i = 0; i < D; i++) du[i] = -u[i]; }\n"
            "    template <class T> __device__ __forceinline__ static void vjp_u(const T* u, const T* p, const T* l, T* dl) { for (int i = 0; i < D; i++) dl[i] = -l[i]; }\n"
            "    template <class T> __device__ __forceinline__ static void vjp_p(const T* u, const T* p, const T* l, T* dg) { for (int q = 0; q < P; q++) dg[q] = 0; }\n"
            + ga +
            "    template <class T> __device__ __forceinline__ static void gvjp_u_apply(const T* u, const T* p, const T* l, const T* w, T* dl) {\n"
            "        T s = 0; for (int j = 0; j < M; j++) s += w[j]; for (int i = 0; i < D; i++) dl[i] = p[0] * l[i] * s; }\n"
            "    template <class T> __device__ __forceinline__ static void gvjp_p_apply(const T* u, const T* p, const T* l, const T* w, T* dg) {\n"
            "        T s = 0; for (int j = 0; j < M; j++) s += w[j]; for (int q = 0; q < P; q++) dg[q] = 0;\n"
            "        for (int i = 0; i < D; i++) dg[0] += u[i] * l[i] * s; }\n};\n")


@pytest.mark.parametrize("D,P,M,g_apply,msg", [(2, 2, 5, True, "1 <= M <= 4"), (2, 2, 0, True, "1 <= M <= 4"), (5, 2, 2, True, "1 <= D <= 4"),
                                               (2, 9, 2, True, "1 <= P <= 8"), (2, 2, 2, False, "g_apply")],
                         ids=["M5", "M0", "D5", "P9", "no_g_apply"])
def test_out_of_range_or_incomplete_family_does_not_compile(tmp_path, D, P, M, g_apply, msg):
    hdr = tmp_path / "probe.cuh"
    hdr.write_text(_family(D, P, M, g_apply))
    with pytest.raises(RuntimeError) as e:
        b.build_family_plugin(str(hdr), "Probe", "probe", out=str(tmp_path / "libprobe.so"), sde=True, noise="general")
    assert msg in str(e.value)


def test_builder_options():
    with pytest.raises(ValueError):
        b.build_family_plugin("x.cuh", "X", "x", noise="general")              # general noise is an SDE shape
    with pytest.raises(ValueError):
        b.build_family_plugin("x.cuh", "X", "x", sde=True, noise="mixing")


FORGED = """#include "handle.h"
namespace {{ int fwd(b200adj::Handle*, const b200adj::SdeFwdArgs&) {{ return 0; }} int rev(b200adj::Handle*, const b200adj::SdeRevArgs&) {{ return 0; }} }}
extern "C" const b200adj::FamilyVTable* b200adj_family_plugin(void) {{
    using namespace b200adj;
    static const FamilyVTable vt = {{B200ADJ_PLUGIN_ABI, {d}, 2, "forged", nullptr, nullptr, nullptr, nullptr, nullptr, nullptr, nullptr, nullptr, 0,
                                    {m}, {kind}, &fwd, &rev}};
    return &vt;
}}
"""


@pytest.mark.parametrize("d,m,kind,code,msg", [(2, 3, "B200ADJ_NOISE_DIAGONAL", -2, "M == D"), (3, 2, "B200ADJ_NOISE_DIAGONAL", -2, "M == D"),
                                               (2, 5, "B200ADJ_NOISE_GENERAL", -2, "M == D"), (2, 2, "B200ADJ_NOISE_NONE", -2, "M == D"),
                                               (2, 0, "B200ADJ_NOISE_DIAGONAL", -1, "no noise")],
                         ids=["diag_m3_d2", "diag_m2_d3", "general_m5", "sde_without_kind", "ode_with_kind"])
def test_registry_refuses_a_noise_shape_outside_the_kernels(tmp_path, d, m, kind, code, msg):
    src = tmp_path / "forged.cu"
    src.write_text(FORGED.format(d=d, m=m, kind=kind))
    so = tmp_path / f"libforged_{d}_{m}.so"
    res = subprocess.run([_lib.nvcc_path(), "-gencode", "arch=compute_90a,code=sm_90a", "-O3", "-std=c++17", "-Xcompiler", "-fPIC",
                          "-shared", "-I", _lib._CSRC, str(src), "-o", str(so)], capture_output=True, text=True)
    assert res.returncode == 0, res.stderr[-3000:]
    with pytest.raises(_lib.B200AdjError) as e:
        b.register_family(str(so))
    assert e.value.code == code and msg in str(e.value)


def _prob(name, d, P, proto=None, tspan=(0.0, 1.0)):
    return b.EnsembleProblem(b.SDEProblem(name, np.ones(d), tspan, np.full(P, 0.1), noise_rate_prototype=proto), u0s=np.ones((d, 4)))


def test_noise_rate_prototype_shape_is_checked_before_a_handle_exists():
    _register("sde_nonsquare")
    for proto in (np.zeros((2, 3)), np.zeros((3, 3)), np.zeros(3), np.zeros((3, 2, 1))):
        with pytest.raises(ValueError, match="noise_rate_prototype"):
            b.solve(_prob("sde_nonsquare", 3, 2, proto), b.EulerHeun(dt=0.1), b.EnsembleB200(device=0), saveat=0.5)
    _check_noise_rate_prototype(b.SDEProblem("sde_nonsquare", np.ones(3), (0.0, 1.0), noise_rate_prototype=np.zeros((3, 2))), 3, 2)
    with pytest.raises(ValueError, match="not a general-noise"):          # a diagonal family takes none
        b.solve(_prob("sde_lv", 2, 6, np.zeros((2, 2))), b.EulerHeun(dt=0.1), b.EnsembleB200(device=0), saveat=0.5)


def test_em_backsolve_on_general_noise_is_refused_before_a_handle_exists():
    _register("sde_roessler")
    for sa in (b.BacksolveAdjoint(), b.B200Adjoint(b.BacksolveAdjoint(checkpointing=False))):
        with pytest.raises(NotImplementedError, match="EM \\+ BacksolveAdjoint"):
            b.solve(_prob("sde_roessler", 2, 4, np.zeros((2, 2))), b.EM(dt=0.1), b.EnsembleB200(device=0), saveat=0.5, sensealg=sa)
    for stepper, sa in (("em", b.InterpolatingAdjoint()), ("euler_heun", b.BacksolveAdjoint()), ("em", None)):
        _check_general_noise("sde_roessler", stepper, sa)
    _check_general_noise("sde_lv", "em", b.BacksolveAdjoint())            # diagonal noise: the Ito-transformed drift


def test_noisemixing_is_accepted_for_a_general_family():
    _register("sde_mixing")
    _register("sde_chain3")
    for sa in (b.BacksolveAdjoint(noisemixing=True), b.B200Adjoint(b.InterpolatingAdjoint(noisemixing=True))):
        _check_noise_mixing("sde_mixing", sa)
        with pytest.raises(NotImplementedError, match="noisemixing"):
            _check_noise_mixing("sde_chain3", sa)
