"""ctypes binding of libb200adj.so (include/b200adj.h) and the in-tree build recipe.

The product path has NO CPU fallback: `load()` raises if the CUDA extension is missing, and `Handle` raises
`B200AdjError` on every non-zero status the C ABI returns.
"""
import ctypes as C
import os
import shutil
import subprocess

_PKG = os.path.dirname(os.path.abspath(__file__))
_ROOT = os.path.dirname(_PKG)
_CSRC = os.path.join(_PKG, "csrc")
LIB_PATH = os.environ.get("B200ADJ_LIB", os.path.join(_PKG, "libb200adj.so"))   # env override: tuning experiments only

FAM = {"lv": 0, "lorenz": 1, "robertson": 2, "sde_lv": 3, "mlp": 4, "sde_linear": 5, "ball": 6, "relax": 7}
SA = {"interpolating": 0, "gauss": 1, "quadrature": 2, "backsolve": 3, "gauss_kronrod": 4}
ST = {"tsit5_fixed": 0, "rosenbrock23": 1, "em": 2, "euler_heun": 3, "tsit5_adaptive": 4}
DTYPE = {"f64": 0, "f32": 1, "bf16_f32acc": 2}
COST = {"explicit": 0, "affine": 1}
FLAG_NO_START, FLAG_NO_CHECKPOINTING, FLAG_CKPT_EVERY_STEP, FLAG_STORED_NOISE, FLAG_TRACE, FLAG_NO_ROTATE, FLAG_DENSE_FORWARD, FLAG_NCCL_ALLREDUCE = 1, 2, 4, 8, 16, 32, 64, 128
FLAG_CHECKPOINT_SAVES = 256        # adaptive Tsit5: checkpointed save intervals, re-solved one at a time by the reverse pass
NOISE_NONE, NOISE_DIAGONAL, NOISE_GENERAL = 0, 1, 2
ERR = {0: "OK", -1: "INVALID", -2: "UNSUPPORTED", -3: "NO_DEVICE", -4: "CUDA", -5: "STATE", -6: "OOM"}

EXPORTS = ["b200adj_create", "b200adj_forward", "b200adj_reverse", "b200adj_set_reverse_options", "b200adj_set_tolerances", "b200adj_set_continuous_cost", "b200adj_set_cost_family", "b200adj_register_family", "b200adj_family_info", "b200adj_set_events", "b200adj_set_event_param_shift", "b200adj_set_continuous_callback", "b200adj_set_continuous_callback_params", "b200adj_event_times", "b200adj_family_conditions", "b200adj_family_noise", "b200adj_family_noise_kind", "b200adj_set_family_events", "b200adj_event_flags", "b200adj_get_noise", "b200adj_set_stream",
           "b200adj_synchronize", "b200adj_launch_count", "b200adj_device_bytes", "b200adj_get_step_counts", "b200adj_get_block_trace", "b200adj_destroy",
           "b200adj_last_error", "b200adj_version", "b200adj_sizeof_cfg",
           "b200adj_comm_unique_id", "b200adj_comm_init", "b200adj_comm_init_all", "b200adj_comm_allreduce", "b200adj_comm_size", "b200adj_comm_is_fused"]


class B200AdjError(RuntimeError):
    def __init__(self, code, msg):
        super().__init__(f"b200adj error {code} ({ERR.get(code, '?')}): {msg}")
        self.code = code


class Cfg(C.Structure):
    _fields_ = [
        ("rhs_family", C.c_int32), ("sensealg", C.c_int32), ("stepper", C.c_int32), ("dtype", C.c_int32),
        ("d", C.c_int32), ("P", C.c_int32), ("m", C.c_int32), ("K", C.c_int32),
        ("N", C.c_int64),
        ("t0", C.c_double), ("t1", C.c_double), ("dt", C.c_double),
        ("abstol", C.c_double), ("reltol", C.c_double),
        ("quad_abstol", C.c_double), ("quad_reltol", C.c_double),
        ("saveat", C.POINTER(C.c_double)),
        ("shared_p", C.c_int32), ("buffers_on_device", C.c_int32), ("device", C.c_int32), ("cost_kind", C.c_int32),
        ("cost_a", C.c_double), ("cost_b", C.c_double),
        ("seed", C.c_uint64), ("traj_offset", C.c_int64),
        ("checkpoint_every", C.c_int32), ("flags", C.c_uint32), ("mlp_hidden", C.c_int32), ("block_threads", C.c_int32),
        ("max_steps", C.c_int32), ("reserved0", C.c_int32),
    ]


def nvcc_path():
    return shutil.which("nvcc") or "/usr/local/cuda/bin/nvcc"


def build(force=False, verbose=False):
    """Compile csrc/*.cu for sm_90a into scimlsensitivity.jl_b200/libb200adj.so (in-tree, next to the package)."""
    from concurrent.futures import ThreadPoolExecutor
    srcs = [os.path.join(_CSRC, f) for f in sorted(os.listdir(_CSRC)) if f.endswith((".cu", ".cuh", ".inc", ".h"))]
    srcs.append(os.path.join(_ROOT, "include", "b200adj.h"))
    if not force and os.path.exists(LIB_PATH) and all(os.path.getmtime(LIB_PATH) >= os.path.getmtime(s) for s in srcs):
        return LIB_PATH
    cus = [s for s in srcs if s.endswith(".cu")]
    objdir = os.path.join(_PKG, "build")
    os.makedirs(objdir, exist_ok=True)
    flags = ["-gencode", "arch=compute_90a,code=sm_90a", "-lineinfo", "-O3", "-std=c++17", "-Xcompiler", "-fPIC", "-Xptxas", "-v"]

    def deps(cu):
        """headers a translation unit includes, transitively (quoted includes inside csrc/ and include/)"""
        seen, todo = set(), [cu]
        while todo:
            f = todo.pop()
            if f in seen or not os.path.exists(f):
                continue
            seen.add(f)
            for line in open(f):
                if line.startswith('#include "'):
                    todo.append(os.path.normpath(os.path.join(os.path.dirname(f), line.split('"')[1])))
        return seen

    def compile_one(cu):
        obj = os.path.join(objdir, os.path.basename(cu)[:-3] + ".o")
        log = obj[:-2] + ".log"
        if not force and os.path.exists(obj) and os.path.exists(log) and all(os.path.getmtime(obj) >= os.path.getmtime(d) for d in deps(cu)):
            return obj, 0, open(log).read()
        res = subprocess.run([nvcc_path()] + flags + ["-c", cu, "-o", obj], capture_output=True, text=True)
        out = res.stdout + res.stderr
        with open(log, "w") as f:
            f.write(out)
        return obj, res.returncode, out

    # heaviest translation units first (the fixed-step and adaptive Tsit5 reverse kernels dominate the build)
    order = sorted(cus, key=lambda c: 0 if "disp_fixed" in c else 1 if "disp_t5a" in c else 2)
    with ThreadPoolExecutor(max_workers=min(len(order), os.cpu_count() or 4)) as ex:
        results = list(ex.map(compile_one, order))
    with open(os.path.join(_PKG, "ptxas.log"), "w") as f:
        f.write("".join(r[2] for r in results))
    bad = [r for r in results if r[1] != 0]
    if bad:
        raise RuntimeError("nvcc failed:\n" + "\n".join(r[2][-4000:] for r in bad))
    # host link with g++ (no -rdc code: nvcc's device-link step would only add an empty default-arch sm_52 stub cubin)
    cuda_lib = os.path.join(os.path.dirname(os.path.dirname(os.path.realpath(nvcc_path()))), "lib64")
    res = subprocess.run(["g++", "-shared", "-o", LIB_PATH] + [r[0] for r in results] + ["-L" + cuda_lib, "-lcudart_static", "-lrt", "-lpthread", "-ldl"],
                         capture_output=True, text=True)
    if res.returncode != 0:
        raise RuntimeError("link failed:\n" + res.stderr[-4000:])
    if verbose:
        print("".join(r[2] for r in results)[-2000:])
    return LIB_PATH


_lib = None


def load():
    global _lib
    if _lib is None:
        if not os.path.exists(LIB_PATH):
            raise ImportError(f"{LIB_PATH} is missing: run `python -c 'import __graft_entry__ as g; g.build()'` "
                              "(the engine has no CPU fallback)")
        lib = C.CDLL(LIB_PATH)
        lib.b200adj_create.argtypes = [C.POINTER(Cfg), C.POINTER(C.c_void_p)]
        lib.b200adj_create.restype = C.c_int32
        lib.b200adj_forward.argtypes = [C.c_void_p] * 6
        lib.b200adj_forward.restype = C.c_int32
        lib.b200adj_reverse.argtypes = [C.c_void_p] * 4
        lib.b200adj_reverse.restype = C.c_int32
        lib.b200adj_set_reverse_options.argtypes = [C.c_void_p, C.c_int32, C.c_int32, C.c_double, C.c_double, C.c_uint32,
                                                    C.c_int32, C.c_void_p]
        lib.b200adj_set_reverse_options.restype = C.c_int32
        lib.b200adj_set_tolerances.argtypes = [C.c_void_p, C.c_double, C.c_double, C.c_double, C.c_double]
        lib.b200adj_set_tolerances.restype = C.c_int32
        lib.b200adj_set_continuous_cost.argtypes = [C.c_void_p, C.c_int32, C.c_double, C.c_double]
        lib.b200adj_set_continuous_cost.restype = C.c_int32
        lib.b200adj_set_cost_family.argtypes = [C.c_void_p, C.c_int32, C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p]
        lib.b200adj_set_cost_family.restype = C.c_int32
        lib.b200adj_register_family.argtypes = [C.c_char_p, C.POINTER(C.c_int32)]
        lib.b200adj_register_family.restype = C.c_int32
        lib.b200adj_family_info.argtypes = [C.c_int32, C.POINTER(C.c_int32), C.POINTER(C.c_int32), C.POINTER(C.c_char_p)]
        lib.b200adj_family_info.restype = C.c_int32
        lib.b200adj_set_events.argtypes = [C.c_void_p, C.c_int32, C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p]
        lib.b200adj_set_events.restype = C.c_int32
        lib.b200adj_set_continuous_callback.argtypes = [C.c_void_p, C.c_int32, C.c_int32, C.c_double, C.c_int32, C.c_void_p, C.c_void_p,
                                                        C.c_int32, C.c_int32, C.c_double, C.c_int32]
        lib.b200adj_set_continuous_callback.restype = C.c_int32
        lib.b200adj_set_event_param_shift.argtypes = [C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p]
        lib.b200adj_set_event_param_shift.restype = C.c_int32
        lib.b200adj_set_continuous_callback_params.argtypes = [C.c_void_p, C.c_int32, C.c_double, C.c_int32, C.c_int32, C.c_double, C.c_int32, C.c_double]
        lib.b200adj_set_continuous_callback_params.restype = C.c_int32
        lib.b200adj_event_times.argtypes = [C.c_void_p, C.c_void_p, C.c_void_p]
        lib.b200adj_event_times.restype = C.c_int32
        lib.b200adj_family_conditions.argtypes = [C.c_int32, C.POINTER(C.c_int32)]
        lib.b200adj_family_conditions.restype = C.c_int32
        lib.b200adj_family_noise.argtypes = [C.c_int32, C.POINTER(C.c_int32)]
        lib.b200adj_family_noise.restype = C.c_int32
        lib.b200adj_family_noise_kind.argtypes = [C.c_int32, C.POINTER(C.c_int32)]
        lib.b200adj_family_noise_kind.restype = C.c_int32
        lib.b200adj_set_family_events.argtypes = [C.c_void_p, C.c_int32, C.c_int32, C.c_void_p, C.c_int32]
        lib.b200adj_set_family_events.restype = C.c_int32
        lib.b200adj_event_flags.argtypes = [C.c_void_p, C.c_void_p]
        lib.b200adj_event_flags.restype = C.c_int32
        lib.b200adj_get_noise.argtypes = [C.c_void_p, C.c_void_p]
        lib.b200adj_get_noise.restype = C.c_int32
        lib.b200adj_set_stream.argtypes = [C.c_void_p, C.c_void_p]
        lib.b200adj_set_stream.restype = C.c_int32
        lib.b200adj_synchronize.argtypes = [C.c_void_p]
        lib.b200adj_synchronize.restype = C.c_int32
        lib.b200adj_launch_count.argtypes = [C.c_void_p]
        lib.b200adj_launch_count.restype = C.c_int64
        lib.b200adj_device_bytes.argtypes = [C.c_void_p, C.POINTER(C.c_int64)]
        lib.b200adj_device_bytes.restype = C.c_int32
        lib.b200adj_get_step_counts.argtypes = [C.c_void_p, C.c_void_p, C.c_void_p]
        lib.b200adj_get_step_counts.restype = C.c_int32
        lib.b200adj_get_block_trace.argtypes = [C.c_void_p, C.c_void_p, C.POINTER(C.c_int32)]
        lib.b200adj_get_block_trace.restype = C.c_int32
        lib.b200adj_destroy.argtypes = [C.c_void_p]
        lib.b200adj_destroy.restype = C.c_int32
        lib.b200adj_comm_unique_id.argtypes = [C.c_void_p]
        lib.b200adj_comm_unique_id.restype = C.c_int32
        lib.b200adj_comm_init.argtypes = [C.c_void_p, C.c_int32, C.c_int32, C.c_void_p]
        lib.b200adj_comm_init.restype = C.c_int32
        lib.b200adj_comm_init_all.argtypes = [C.POINTER(C.c_void_p), C.c_int32]
        lib.b200adj_comm_init_all.restype = C.c_int32
        lib.b200adj_comm_allreduce.argtypes = [C.c_void_p, C.c_void_p, C.c_int64]
        lib.b200adj_comm_allreduce.restype = C.c_int32
        lib.b200adj_comm_is_fused.argtypes = [C.c_void_p]
        lib.b200adj_comm_is_fused.restype = C.c_int32
        lib.b200adj_comm_size.argtypes = [C.c_void_p, C.POINTER(C.c_int32), C.POINTER(C.c_int32)]
        lib.b200adj_comm_size.restype = C.c_int32
        lib.b200adj_last_error.argtypes = [C.c_void_p]
        lib.b200adj_last_error.restype = C.c_char_p
        lib.b200adj_version.restype = C.c_uint32
        lib.b200adj_sizeof_cfg.restype = C.c_uint32
        if lib.b200adj_sizeof_cfg() != C.sizeof(Cfg):
            raise ImportError(f"b200adj_cfg layout mismatch: C {lib.b200adj_sizeof_cfg()} vs ctypes {C.sizeof(Cfg)}")
        _lib = lib
    return _lib


def _addr(x):
    """Raw address of a numpy array, a torch tensor, an int, or None."""
    if x is None:
        return None
    if isinstance(x, int):
        return x
    if hasattr(x, "data_ptr"):
        return x.data_ptr()
    return x.ctypes.data


def family_conditions(family_id):
    """Number of conditions compiled into a family (0: none)."""
    nc = C.c_int32()
    rc = load().b200adj_family_conditions(int(family_id), C.byref(nc))
    if rc != 0:
        raise B200AdjError(rc, f"unknown family id {family_id}")
    return nc.value


def family_noise(family_id):
    """Number of Wiener processes of a family: m = d for a diagonal-noise SDE family, the M of a general-noise one, 0 for an
    ODE family."""
    m = C.c_int32()
    rc = load().b200adj_family_noise(int(family_id), C.byref(m))
    if rc != 0:
        raise B200AdjError(rc, f"unknown family id {family_id}")
    return m.value


def family_noise_kind(family_id):
    """Shape of a family's noise term: NOISE_NONE (ODE family), NOISE_DIAGONAL (g .* dW) or NOISE_GENERAL (G dW, G of size d x m)."""
    k = C.c_int32()
    rc = load().b200adj_family_noise_kind(int(family_id), C.byref(k))
    if rc != 0:
        raise B200AdjError(rc, f"unknown family id {family_id}")
    return k.value


def comm_unique_id():
    """128-byte NCCL unique id (call on rank 0, broadcast over the host's own channel)."""
    buf = C.create_string_buffer(128)
    rc = load().b200adj_comm_unique_id(buf)
    if rc != 0:
        raise B200AdjError(rc, "b200adj_comm_unique_id failed (libnccl.so.2 not loadable?)")
    return buf.raw


def comm_init_all(handles):
    """One process driving several GPUs: the handles (one per device) become ranks 0..n-1 of one NCCL communicator.
    Their reverse() calls must then run concurrently (one host thread per handle)."""
    arr = (C.c_void_p * len(handles))(*[h._h for h in handles])
    rc = load().b200adj_comm_init_all(arr, len(handles))
    if rc != 0:
        raise B200AdjError(rc, load().b200adj_last_error(handles[0]._h).decode())


class Handle:
    """Owner of one b200adj handle (one GPU, one ensemble shard)."""

    def __init__(self, cfg: Cfg, saveat):
        import numpy as np
        self._lib = load()
        self._saveat = np.ascontiguousarray(saveat, dtype=np.float64)
        cfg.K = len(self._saveat)
        cfg.saveat = self._saveat.ctypes.data_as(C.POINTER(C.c_double))
        self.cfg = cfg
        self._h = C.c_void_p()
        rc = self._lib.b200adj_create(C.byref(cfg), C.byref(self._h))
        if rc != 0:
            raise B200AdjError(rc, self._lib.b200adj_last_error(None).decode())

    def _check(self, rc):
        if rc != 0:
            raise B200AdjError(rc, self._lib.b200adj_last_error(self._h).decode())

    def forward(self, u0, p, saved=None, status=None, dW=None):
        self._check(self._lib.b200adj_forward(self._h, _addr(u0), _addr(p), _addr(dW), _addr(saved), _addr(status)))

    def reverse(self, dLdu, du0, dp):
        self._check(self._lib.b200adj_reverse(self._h, _addr(dLdu), _addr(du0), _addr(dp)))

    def set_reverse_options(self, sensealg, cost_kind, cost_a, cost_b, flags, t=None):
        import numpy as np
        if t is None:
            K, tp = -1, None
        else:
            self._t = np.ascontiguousarray(t, dtype=np.float64)
            K, tp = len(self._t), self._t.ctypes.data
        self._check(self._lib.b200adj_set_reverse_options(self._h, sensealg, cost_kind, cost_a, cost_b, flags, K, tp))

    def set_tolerances(self, adj_abstol=0.0, adj_reltol=0.0, quad_abstol=0.0, quad_reltol=0.0):
        self._check(self._lib.b200adj_set_tolerances(self._h, adj_abstol, adj_reltol, quad_abstol, quad_reltol))

    def set_continuous_cost(self, enabled, a=0.0, b=0.0):
        self._check(self._lib.b200adj_set_continuous_cost(self._h, int(bool(enabled)), float(a), float(b)))

    def set_cost_family(self, which, a=None, b=None, c=None, e=None):
        """Per-component coefficients of the named cost family (which = 0 discrete, 1 continuous): dgdu = a .* u + b,
        dgdp = c .* p + e; None keeps (a, b) / zeroes (c, e)."""
        import numpy as np
        arrs = [None if x is None else np.ascontiguousarray(x, dtype=np.float64).reshape(-1) for x in (a, b, c, e)]
        self._check(self._lib.b200adj_set_cost_family(self._h, int(which), *[None if x is None else x.ctypes.data for x in arrs]))

    def set_events(self, times, scale, shift, pscale=None, pshift=None):
        """Preset-time events u <- scale[e] * u + shift[e] (and optionally p <- pscale[e] * p + pshift[e]) at times[e]
        (host arrays; empty = none)."""
        import numpy as np
        t = np.ascontiguousarray(times, dtype=np.float64).reshape(-1)
        E = len(t)
        sc = np.ascontiguousarray(scale, dtype=np.float64).reshape(E, -1) if E else None      # E = 0 removes the events
        sh = np.ascontiguousarray(shift, dtype=np.float64).reshape(E, -1) if E else None
        ps = pc = None
        if pscale is not None and E:
            ps = np.ascontiguousarray(pscale, dtype=np.float64).reshape(E, -1)
            pc = np.ascontiguousarray(pshift, dtype=np.float64).reshape(E, -1)
        self._check(self._lib.b200adj_set_events(self._h, E, t.ctypes.data if E else None, sc.ctypes.data if E else None,
                                                 sh.ctypes.data if E else None, None if ps is None else ps.ctypes.data,
                                                 None if pc is None else pc.ctypes.data))

    def set_event_param_shift(self, comp, param, coef):
        """u[comp[e]] += coef[e] * p[param[e]] at preset event e (after set_events; comp = None removes)."""
        import numpy as np
        if comp is None:
            self._check(self._lib.b200adj_set_event_param_shift(self._h, None, None, None))
            return
        ac = np.ascontiguousarray(comp, dtype=np.int32).reshape(-1)
        ak = np.ascontiguousarray(param, dtype=np.int32).reshape(-1)
        af = np.ascontiguousarray(coef, dtype=np.float64).reshape(-1)
        self._check(self._lib.b200adj_set_event_param_shift(self._h, ac.ctypes.data, ak.ctypes.data, af.ctypes.data))

    def set_continuous_callback(self, idx, level=0.0, direction=-1, scale=None, shift=None, pcomp=-1, pparam=0, psign=1.0,
                                max_events=64, enabled=True):
        """State-dependent event: condition u[idx] - level, affine affect (+ u[pcomp] <- psign * p[pparam] * u[pcomp])."""
        import numpy as np
        sc = None if scale is None else np.ascontiguousarray(scale, dtype=np.float64).reshape(-1)
        sh = None if shift is None else np.ascontiguousarray(shift, dtype=np.float64).reshape(-1)
        self._check(self._lib.b200adj_set_continuous_callback(self._h, 1 if enabled else 0, int(idx), float(level), int(direction),
                                                              None if sc is None else sc.ctypes.data, None if sh is None else sh.ctypes.data,
                                                              int(pcomp), int(pparam), float(psign), int(max_events)))

    def set_continuous_callback_params(self, lparam=-1, lcoef=0.0, acomp=-1, aparam=0, acoef=0.0, qcomp=-1, qcoef=1.0):
        """Parameter-dependent level (level += lcoef * p[lparam]), additive parameter affect (u[acomp] += acoef * p[aparam]),
        quadratic affect (u[qcomp] <- qcoef * u[qcomp]^2)."""
        self._check(self._lib.b200adj_set_continuous_callback_params(self._h, int(lparam), float(lcoef), int(acomp), int(aparam), float(acoef),
                                                                     int(qcomp), float(qcoef)))

    def event_times(self, N, max_events):
        """-> (counts[N], times[max_events, N]) found by the last forward pass."""
        import numpy as np
        counts = np.zeros(N, dtype=np.int32)
        times = np.zeros((max_events, N), dtype=np.float64)
        self._check(self._lib.b200adj_event_times(self._h, counts.ctypes.data, times.ctypes.data))
        return counts, times

    def set_family_events(self, nc, direction, max_events=64, enabled=True):
        """State-dependent event with the conditions and affect compiled into the family; direction[nc] in {-1, 0, 1}."""
        import numpy as np
        dr = np.ascontiguousarray(direction, dtype=np.int32).reshape(-1)
        self._check(self._lib.b200adj_set_family_events(self._h, 1 if enabled else 0, int(nc), dr.ctypes.data if len(dr) else None,
                                                        int(max_events)))

    def event_flags(self, N, max_events):
        """-> words[max_events, N] (int32) of the last forward pass: bit 2c = condition c fired, bit 2c + 1 = upwards."""
        import numpy as np
        ev = np.zeros((max_events, N), dtype=np.int32)
        self._check(self._lib.b200adj_event_flags(self._h, ev.ctypes.data))
        return ev

    def step_counts(self, fwd, rev):
        self._check(self._lib.b200adj_get_step_counts(self._h, _addr(fwd), _addr(rev)))

    def get_noise(self, out):
        self._check(self._lib.b200adj_get_noise(self._h, _addr(out)))

    def block_trace(self):
        """[nblocks, 3] uint64: (SM id, start ns, end ns) of every block of the last reverse launch (FLAG_TRACE)."""
        import numpy as np
        n = C.c_int32()
        self._check(self._lib.b200adj_get_block_trace(self._h, None, C.byref(n)))
        out = np.zeros((n.value, 3), dtype=np.uint64)
        self._check(self._lib.b200adj_get_block_trace(self._h, out.ctypes.data, C.byref(n)))
        return out

    def comm_init(self, nranks, rank, unique_id):
        """Attach this handle to an NCCL communicator of `nranks` handles (one per GPU); b200adj_reverse then sums dp over
        the ranks itself.  unique_id: the 128 bytes of comm_unique_id() from rank 0."""
        buf = C.create_string_buffer(bytes(unique_id), 128) if unique_id is not None else None
        self._check(self._lib.b200adj_comm_init(self._h, int(nranks), int(rank), buf))

    def comm_allreduce(self, buf, count):
        self._check(self._lib.b200adj_comm_allreduce(self._h, _addr(buf), int(count)))

    @property
    def comm_is_fused(self):
        return bool(self._lib.b200adj_comm_is_fused(self._h))

    @property
    def comm_size(self):
        n, r = C.c_int32(), C.c_int32()
        self._check(self._lib.b200adj_comm_size(self._h, C.byref(n), C.byref(r)))
        return n.value, r.value

    def set_stream(self, stream_ptr):
        self._check(self._lib.b200adj_set_stream(self._h, stream_ptr))

    def synchronize(self):
        self._check(self._lib.b200adj_synchronize(self._h))

    @property
    def launch_count(self):
        return int(self._lib.b200adj_launch_count(self._h))

    def device_bytes(self):
        """Device memory the handle owns now, in bytes."""
        n = C.c_int64()
        self._check(self._lib.b200adj_device_bytes(self._h, C.byref(n)))
        return n.value

    def close(self):
        if self._h:
            self._lib.b200adj_destroy(self._h)
            self._h = C.c_void_p()

    def __del__(self):
        try:
            self.close()
        except Exception:
            pass
