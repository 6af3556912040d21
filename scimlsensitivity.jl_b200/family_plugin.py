"""User RHS families as plug-ins of libb200adj.so (SURVEY.md 8f rank 4).

The reference lets a user hand `ODEFunction(f; vjp, vjp_p, jac, paramjac)` to the adjoint (src/derivative_wrappers.jl:284-359,
test/Core3/user_vjp.jl:14-38).  The device equivalent: write ONE struct in a CUDA header with the shape of csrc/families.cuh
(device functions f, vjp_u, vjp_p, optionally jac / djac / dvjp_p), build it into a plug-in with `build_family_plugin` (nvcc
instantiates the library's own kernel templates for it -- no .cu file of the library is edited) and `register_family` it; the
name is then usable wherever "lv" / "lorenz" are.

    python -m scimlsensitivity_jl_b200.family_plugin my_family.cuh VanDerPol vanderpol [--jac] [-o libfam_vanderpol.so]
"""
import ctypes as C
import os
import subprocess
import sys
import tempfile

from . import _lib
from .problems import FAMILIES


def build_family_plugin(header, struct, name, out=None, has_jac=False, verbose=False):
    """Compile `struct` of the CUDA header `header` into a family plug-in (shared library); returns its path."""
    header = os.path.abspath(header)
    out = os.path.abspath(out or os.path.join(os.path.dirname(header), f"libb200fam_{name}.so"))
    if os.path.exists(out) and os.path.getmtime(out) >= max(os.path.getmtime(header), os.path.getmtime(_lib.LIB_PATH)):
        return out
    pkg = os.path.dirname(_lib.LIB_PATH)
    with tempfile.TemporaryDirectory() as tmp:
        src = os.path.join(tmp, f"fam_{name}.cu")
        with open(src, "w") as f:
            f.write(f'#include "{header}"\n#define B200ADJ_FAMILY {struct}\n#define B200ADJ_FAMILY_NAME "{name}"\n')
            if has_jac:
                f.write("#define B200ADJ_FAMILY_HAS_JAC 1\n")
            f.write('#include "family_plugin.inc"\n')
        cmd = [_lib.nvcc_path(), "-gencode", "arch=compute_90a,code=sm_90a", "-lineinfo", "-O3", "-std=c++17", "-Xcompiler", "-fPIC",
               "-shared", "-I", _lib._CSRC, src, "-o", out, "-L", pkg, "-l:" + os.path.basename(_lib.LIB_PATH), "-Xlinker", "-rpath", "-Xlinker", pkg]
        res = subprocess.run(cmd, capture_output=True, text=True)
        if res.returncode != 0:
            raise RuntimeError("nvcc failed building the family plug-in:\n" + res.stderr[-4000:])
        if verbose:
            print(res.stderr[-2000:])
    return out


def register_family(plugin_path, name=None):
    """Load a family plug-in; afterwards `name` (default: the plug-in's own) is a valid RHS family.  Returns (id, d, P)."""
    lib = _lib.load()
    fid = C.c_int32()
    rc = lib.b200adj_register_family(os.path.abspath(plugin_path).encode(), C.byref(fid))
    if rc != 0:
        raise _lib.B200AdjError(rc, lib.b200adj_last_error(None).decode())
    d, P, nm = C.c_int32(), C.c_int32(), C.c_char_p()
    lib.b200adj_family_info(fid.value, C.byref(d), C.byref(P), C.byref(nm))
    name = name or nm.value.decode()
    _lib.FAM[name] = fid.value
    FAMILIES[name] = (d.value, P.value, 0)
    return fid.value, d.value, P.value


if __name__ == "__main__":
    import argparse
    ap = argparse.ArgumentParser(description=__doc__.split("\n")[0])
    ap.add_argument("header"); ap.add_argument("struct"); ap.add_argument("name")
    ap.add_argument("--jac", action="store_true", help="the struct also has jac / djac / dvjp_p: build the Rosenbrock23 kernels")
    ap.add_argument("-o", "--out", default=None)
    a = ap.parse_args()
    print(build_family_plugin(a.header, a.struct, a.name, a.out, a.jac, verbose=True))
