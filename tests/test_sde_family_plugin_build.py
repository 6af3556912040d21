"""SDE family plug-ins without a GPU (nvcc cross-compiles, a plug-in registers without touching the device).

* The seam: SdeLotkaVolterra and SdeLinear2 built as plug-ins straight from the library's own csrc/families.cuh have, kernel
  for kernel, the registers, stack, shared and local memory (spills) of the library's instantiations of the same templates
  (cuobjdump -res-usage): the plug-in path runs the library's hot path, not a variant of it.
* The registry: b200adj_family_noise of every built-in family and of the example plug-ins, FAMILIES[name] = (d, P, m).
* A plug-in built against headers whose SdeRevArgs differs is refused by the ABI tag.
* noisemixing = true on a plug-in SDE family raises on the host before any handle exists.
"""
import os
import re
import shutil
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
from scimlsensitivity_jl_b200.problems import FAMILY_CONDITIONS

FAMILIES_CUH = os.path.join(_lib._CSRC, "families.cuh")
EXAMPLES = os.path.join(ROOT, "examples")


def _cuobjdump():
    return os.path.join(os.path.dirname(_lib.nvcc_path()), "cuobjdump")


def _res_usage(so):
    """{kernel symbol: 'REG:.. STACK:.. SHARED:.. LOCAL:..'} of the SDE kernels in a shared library"""
    out = subprocess.run([_cuobjdump(), "-res-usage", so], capture_output=True, text=True, check=True).stdout
    res, name = {}, None
    for line in out.splitlines():
        m = re.match(r"\s*Function (\S+):", line)
        if m:
            name = m.group(1)
            continue
        if name and "REG:" in line:
            if "sde_" in name:
                res[name] = " ".join(re.findall(r"(?:REG|STACK|SHARED|LOCAL):\d+", line))
            name = None
    return res


@pytest.fixture(scope="module")
def seam_plugins(tmp_path_factory):
    tmp = tmp_path_factory.mktemp("sde_seam")
    return {struct: b.build_family_plugin(FAMILIES_CUH, struct, name, out=str(tmp / f"libb200fam_{name}.so"), sde=True)
            for struct, name in (("SdeLotkaVolterra", "sde_lv_seam"), ("SdeLinear2", "sde_linear_seam"))}


@pytest.mark.parametrize("struct", ["SdeLotkaVolterra", "SdeLinear2"])
def test_plugin_kernels_have_the_library_resources(seam_plugins, struct):
    lib = _res_usage(_lib.LIB_PATH)
    plug = _res_usage(seam_plugins[struct])
    mine = {k: v for k, v in lib.items() if f"{len(struct)}{struct}I" in k}
    # forward: EM / EulerHeun x shared / per-member p; reverse: (EM Backsolve on the Ito drift, EulerHeun Backsolve,
    # Interpolating x EM / EulerHeun) x shared / per-member p x affine / explicit cost
    assert len(plug) == 4 + 16 and set(plug) == set(mine), set(plug) ^ set(mine)
    for k in plug:
        assert plug[k] == mine[k], (k, plug[k], mine[k])


def test_family_noise_and_registry():
    expect = {"lv": 0, "lorenz": 0, "robertson": 0, "sde_lv": 2, "mlp": 0, "sde_linear": 2, "ball": 0, "relax": 0}
    for name, m in expect.items():
        assert _lib.family_noise(_lib.FAM[name]) == m
    for bad in (8, 99, 100 + 10_000, -1):
        with pytest.raises(_lib.B200AdjError) as e:
            _lib.family_noise(bad)
        assert e.value.code == -1
    for struct, name, d, P in (("SdeFoodChain3", "sde_chain3", 3, 6), ("SdeOscillator4", "sde_osc4", 4, 8)):
        so = os.path.join(EXAMPLES, f"libb200fam_{name}.so")
        if not os.path.exists(so):
            pytest.skip("the example plug-ins are built by __graft_entry__.build()")
        fid, d_, P_ = b.register_family(so)
        assert (d_, P_) == (d, P) and fid >= 100
        assert _lib.family_noise(fid) == d and b.FAMILIES[name] == (d, P, d) and FAMILY_CONDITIONS[name] == 0
    vdp = os.path.join(EXAMPLES, "libb200fam_vanderpol.so")
    if os.path.exists(vdp):
        fid, _, _ = b.register_family(vdp)
        assert _lib.family_noise(fid) == 0 and b.FAMILIES["vanderpol"][2] == 0


def test_plugin_built_against_other_headers_is_refused(tmp_path):
    """the same family, built against headers whose SdeRevArgs has one more field: the ABI tag differs"""
    csrc = tmp_path / "pkg" / "csrc"          # the tree's layout: csrc/handle.h includes ../../include/b200adj.h
    shutil.copytree(_lib._CSRC, csrc, ignore=shutil.ignore_patterns("*.so", "*.o", "build", "*.log"))
    shutil.copytree(os.path.join(ROOT, "include"), tmp_path / "include")
    sde = (csrc / "sde_em.cuh").read_text()
    tail = "int64_t N; int32_t S; double h; double cost_a[4], cost_b[4]; uint32_t flags; uint64_t seed; int64_t traj_offset;\n};"
    assert tail in sde
    (csrc / "sde_em.cuh").write_text(sde.replace(tail, tail[:-3] + " double extra;\n};", 1))
    src = tmp_path / "fam.cu"
    src.write_text(f'#include "{FAMILIES_CUH}"\n#define B200ADJ_FAMILY SdeLinear2\n#define B200ADJ_FAMILY_NAME "stale"\n'
                   '#define B200ADJ_FAMILY_SDE 1\n#include "family_plugin.inc"\n')
    so = tmp_path / "libstale.so"
    pkg = os.path.dirname(_lib.LIB_PATH)
    res = subprocess.run([_lib.nvcc_path(), "-gencode", "arch=compute_90a,code=sm_90a", "-O3", "-std=c++17", "-Xcompiler", "-fPIC",
                          "-shared", "-I", str(csrc), str(src), "-o", str(so), "-L", pkg, "-l:" + os.path.basename(_lib.LIB_PATH),
                          "-Xlinker", "-rpath", "-Xlinker", pkg], capture_output=True, text=True)
    assert res.returncode == 0, res.stderr[-3000:]
    with pytest.raises(_lib.B200AdjError) as e:
        b.register_family(str(so))
    assert e.value.code == -1 and "ABI" in str(e.value)


def test_noisemixing_is_refused_for_a_plugin_sde_family():
    so = os.path.join(EXAMPLES, "libb200fam_sde_chain3.so")
    if not os.path.exists(so):
        pytest.skip("the example plug-ins are built by __graft_entry__.build()")
    b.register_family(so)
    prob = b.EnsembleProblem(b.SDEProblem("sde_chain3", np.ones(3), (0.0, 1.0), np.full(6, 0.5)), u0s=np.ones((3, 4)))
    for sa in (b.BacksolveAdjoint(noisemixing=True), b.B200Adjoint(b.InterpolatingAdjoint(noisemixing=True))):
        with pytest.raises(NotImplementedError, match="noisemixing"):
            b.solve(prob, b.EM(dt=0.1), b.EnsembleB200(device=0), saveat=0.5, sensealg=sa)
