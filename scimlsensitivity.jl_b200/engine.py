"""Host-side driver of one device handle: buffer plumbing (numpy host buffers or torch CUDA tensors), cfg assembly.

PyTorch is used here only for device memory and streams (and torch.distributed in distributed.py); all arithmetic
is in libb200adj.so.
"""
import numpy as np

from . import _lib
from .problems import FAMILIES, FAMILY_CONDITIONS, AffineCost, ParamAffine, VectorContinuousCallback


def _is_torch(x):
    return hasattr(x, "data_ptr") and hasattr(x, "device")


class DeviceEnsemble:
    """One ensemble shard on one GPU: forward(u0, p) -> saved, reverse(dLdu) -> (du0, dp)."""

    def __init__(self, family, sensealg, stepper, N, saveat, tspan, dt, *, shared_p=True, cost=None,
                 on_device=False, device=0, no_start=False, checkpointing=True, ckpt_every_step=False,
                 stored_noise=False, seed=0, traj_offset=0, block_threads=0, abstol=1e-6, reltol=1e-3,
                 quad_abstol=1e-6, quad_reltol=1e-3, dtype="f64", trace=False, max_steps=0, pin_outputs=False,
                 checkpoint_every=1, no_rotate=False, dense_forward=False, nccl_allreduce=False):
        d, P, m = FAMILIES[family]
        cfg = _lib.Cfg()
        cfg.rhs_family, cfg.sensealg, cfg.stepper, cfg.dtype = _lib.FAM[family], _lib.SA[sensealg], _lib.ST[stepper], _lib.DTYPE[dtype]
        cfg.d, cfg.P, cfg.m, cfg.N = d, P, m, int(N)
        cfg.t0, cfg.t1, cfg.dt = float(tspan[0]), float(tspan[1]), float(dt)
        cfg.abstol, cfg.reltol, cfg.quad_abstol, cfg.quad_reltol = abstol, reltol, quad_abstol, quad_reltol
        cfg.shared_p, cfg.buffers_on_device, cfg.device = int(shared_p), int(on_device), int(device)
        if isinstance(cost, AffineCost):
            cfg.cost_kind = _lib.COST["affine"]
            cfg.cost_a, cfg.cost_b = (float(cost.a), float(cost.b)) if cost.is_scalar else (0.0, 0.0)
        else:
            cfg.cost_kind = _lib.COST["explicit"]
        cfg.seed, cfg.traj_offset = int(seed), int(traj_offset)
        cfg.mlp_hidden = 64 if family == "mlp" else 0
        self.dtype = dtype
        self.np_dtype = np.float64 if dtype == "f64" else np.float32      # bf16_f32acc: fp32 buffers at the ABI
        cfg.max_steps = int(max_steps or 0)                  # adaptive handles: per-member step capacity (0 = 4096)
        cfg.checkpoint_every = int(checkpoint_every or 1)    # fixed-step Tsit5: interval checkpointing
        flags = 0
        if no_start:
            flags |= _lib.FLAG_NO_START
        if not checkpointing:
            flags |= _lib.FLAG_NO_CHECKPOINTING
        if ckpt_every_step:
            flags |= _lib.FLAG_CKPT_EVERY_STEP
        if stored_noise:
            flags |= _lib.FLAG_STORED_NOISE
        if trace:
            flags |= _lib.FLAG_TRACE
        if no_rotate:
            flags |= _lib.FLAG_NO_ROTATE
        if dense_forward:
            flags |= _lib.FLAG_DENSE_FORWARD
        if nccl_allreduce:
            flags |= _lib.FLAG_NCCL_ALLREDUCE
        cfg.flags, cfg.block_threads = flags, int(block_threads)
        self.family, self.d, self.P, self.m, self.N, self.K = family, d, P, m, int(N), len(saveat)
        self.shared_p, self.on_device, self.device = bool(shared_p), bool(on_device), int(device)
        self.adaptive = stepper in ("rosenbrock23", "tsit5_adaptive")
        self.events = None
        self.S = 0 if self.adaptive else int(round((cfg.t1 - cfg.t0) / cfg.dt))
        self.saveat = np.ascontiguousarray(saveat, dtype=np.float64)
        # the forward pass keeps the create-time save table; set_reverse(t=...) only re-targets the reverse pass
        self.fwd_saveat, self.fwd_K = self.saveat.copy(), len(self.saveat)
        self.handle = _lib.Handle(cfg, self.saveat)
        if isinstance(cost, AffineCost) and not cost.is_scalar:
            self.handle.set_cost_family(0, np.broadcast_to(np.asarray(cost.a, dtype=np.float64), (d,)), np.broadcast_to(np.asarray(cost.b, dtype=np.float64), (d,)))
        self._keep = []
        self.pin_outputs, self._pinned = bool(pin_outputs), {}
        if self.on_device:
            # device-pointer mode is asynchronous: run on torch's current stream so tensor producers/consumers order
            # correctly with the kernels (host-buffer mode synchronises inside the C ABI instead)
            self.use_current_torch_stream()

    # ---- buffers ----
    def _empty(self, *shape, dtype="real", role=""):
        if self.on_device:
            import torch
            td = torch.int32 if dtype == "i32" else (torch.float64 if self.dtype == "f64" else torch.float32)
            return torch.empty(shape, dtype=td, device=f"cuda:{self.device}")
        npdt = np.int32 if dtype == "i32" else self.np_dtype
        if self.pin_outputs:
            # page-locked result buffers, allocated once per (role, shape) and REUSED by later calls on this handle (true
            # async D2H instead of a staged pageable copy); callers that keep results across calls must copy them.  The role
            # keeps two outputs of one call apart when their shapes coincide (du0 / dp with P == d and per-member p).
            key = (role, tuple(shape), np.dtype(npdt).str)
            if key not in self._pinned:
                import torch
                self._pinned[key] = torch.empty(tuple(shape), dtype=getattr(torch, np.dtype(npdt).name), pin_memory=True)
            return self._pinned[key].numpy()
        return np.empty(shape, dtype=npdt)

    def _prep(self, x, shape):
        if self.on_device:
            import torch
            if not _is_torch(x):
                x = torch.as_tensor(np.ascontiguousarray(x, dtype=self.np_dtype), device=f"cuda:{self.device}")
            x = x.to(dtype=torch.float64 if self.dtype == "f64" else torch.float32).contiguous()
            assert tuple(x.shape) == tuple(shape), (tuple(x.shape), shape)
            return x
        if _is_torch(x):
            x = x.detach().cpu().numpy()
        x = np.ascontiguousarray(x, dtype=self.np_dtype)
        assert x.shape == tuple(shape), (x.shape, shape)
        return x

    def use_current_torch_stream(self):
        import torch
        ptr = torch.cuda.current_stream(self.device).cuda_stream
        self.handle.set_stream(ptr if ptr else 1)          # 0 is the legacy default stream: pass cudaStreamLegacy (0x1)

    # ---- passes ----
    def forward(self, u0, p, dW=None, want_saved=True, want_status=True, saved_out=None):
        u0 = self._prep(u0, (self.d, self.N))
        p = self._prep(p, (self.P,) if self.shared_p else (self.P, self.N))
        if dW is not None:
            dW = self._prep(dW, (self.S, self.m, self.N))
        saved = saved_out if saved_out is not None else (self._empty(self.fwd_K, self.d, self.N, role="saved") if (want_saved and self.fwd_K > 0) else None)
        status = self._empty(self.N, dtype="i32", role="status") if want_status else None
        self._keep = [u0, p, dW]                      # p must stay alive until reverse (device mode reads it in place)
        self.handle.forward(u0, p, saved, status, dW)
        return saved, status

    def reverse(self, dLdu=None, du0_out=None, dp_out=None):
        if dLdu is not None:
            dLdu = self._prep(dLdu, (self.K, self.d, self.N))
        du0 = du0_out if du0_out is not None else self._empty(self.d, self.N, role="du0")
        dp = dp_out if dp_out is not None else (self._empty(self.P, role="dp") if self.shared_p else self._empty(self.P, self.N, role="dp"))
        self.handle.reverse(dLdu, du0, dp)
        return du0, dp

    def set_events(self, times, scale, shift, pscale=None, pshift=None):
        """Preset-time events of the hybrid system (adaptive Tsit5): u <- scale[e] * u + shift[e] and, optionally,
        p <- pscale[e] * p + pshift[e] at times[e]; call before forward()."""
        times = np.asarray(times, dtype=np.float64).reshape(-1)
        E = len(times)
        scale = np.asarray(scale, dtype=np.float64).reshape(E, -1) if E else np.zeros((0, self.d))
        shift = np.asarray(shift, dtype=np.float64).reshape(E, -1) if E else np.zeros((0, self.d))
        if E and (scale.shape[1] != self.d or shift.shape[1] != self.d):
            raise ValueError("events: scale and shift must be [E, d]")
        if (pscale is None) != (pshift is None):
            raise ValueError("events: pscale and pshift come together")
        if pscale is not None and E:
            pscale = np.asarray(pscale, dtype=np.float64).reshape(E, -1)
            pshift = np.asarray(pshift, dtype=np.float64).reshape(E, -1)
            if pscale.shape[1] != self.P or pshift.shape[1] != self.P:
                raise ValueError("events: pscale and pshift must be [E, P]")
        self.handle.set_events(times, scale, shift, pscale, pshift)
        self.events = (times, scale, shift, pscale, pshift)

    def set_event_param_shift(self, comp, param, coef):
        """u[comp[e]] += coef[e] * p[param[e]] at preset event e (the "Dosing example" affect); after set_events."""
        self.handle.set_event_param_shift(comp, param, coef)

    def set_continuous_callback(self, cb):
        """State-dependent event (problems.ContinuousCallback, or problems.VectorContinuousCallback with the conditions and
        affect of the family) of the hybrid system; call before forward().  None removes it."""
        if cb is None:
            self.handle.set_continuous_callback(0, enabled=False)
            self.continuous_callback = None
            return
        if isinstance(cb, VectorContinuousCallback):
            if tuple(cb.save_positions) != (False, False):
                raise NotImplementedError("VectorContinuousCallback: save_positions = (false, false) is the mode carried on the device")
            nc = FAMILY_CONDITIONS.get(self.family, 0)
            self.handle.set_family_events(nc, cb.directions(nc) if nc else np.zeros(0, np.int32), cb.max_events)   # nc = 0: refused
            self.continuous_callback = cb
            return
        if tuple(cb.save_positions) != (False, False):
            raise NotImplementedError("ContinuousCallback: save_positions = (false, false) is the mode carried on the device")
        for name, v in (("scale", cb.scale), ("shift", cb.shift)):
            if v is not None and np.asarray(v).reshape(-1).shape[0] != self.d:
                raise ValueError(f"ContinuousCallback: {name} must have d entries")
        self.handle.set_continuous_callback(cb.idx, cb.level, cb.direction, cb.scale, cb.shift, -1 if cb.p_comp is None else cb.p_comp,
                                            cb.p_param, cb.p_sign, cb.max_events)
        if cb.level_param is not None or cb.add_comp is not None or cb.sq_comp is not None:
            self.handle.set_continuous_callback_params(-1 if cb.level_param is None else cb.level_param, cb.level_coef,
                                                       -1 if cb.add_comp is None else cb.add_comp, cb.add_param, cb.add_coef,
                                                       -1 if cb.sq_comp is None else cb.sq_comp, cb.sq_coef)
        self.continuous_callback = cb

    def event_times(self):
        """-> (counts[N], times[max_events, N]): the event lists found by the last forward pass."""
        return self.handle.event_times(self.N, self.continuous_callback.max_events)

    def event_flags(self):
        """VectorContinuousCallback: -> ev[max_events, NC, N] (int8) of the last forward pass, the `ev` each affect saw:
        +1 / -1 for a condition that fired crossing upwards / downwards, 0 for one that did not; 0 past a member's events."""
        nc = FAMILY_CONDITIONS.get(self.family, 0)
        counts, _ = self.handle.event_times(self.N, self.continuous_callback.max_events)
        words = self.handle.event_flags(self.N, self.continuous_callback.max_events)
        words[np.arange(words.shape[0])[:, None] >= counts[None, :]] = 0
        fired = (words[:, None, :] >> (2 * np.arange(nc))[None, :, None]) & 1
        up = (words[:, None, :] >> (2 * np.arange(nc) + 1)[None, :, None]) & 1
        return (fired * (2 * up - 1)).astype(np.int8)

    def set_reverse(self, sensealg, cost=None, no_start=False, checkpointing=True, ckpt_every_step=False, t=None, dgdp=None):
        """Re-target the next reverse pass (sensealg / cost / save times) without re-running the forward pass.
        dgdp: ParamAffine, the parameter part of the discrete cost (dgdp_discrete)."""
        flags = 0
        if no_start:
            flags |= _lib.FLAG_NO_START
        if not checkpointing:
            flags |= _lib.FLAG_NO_CHECKPOINTING
        if ckpt_every_step:
            flags |= _lib.FLAG_CKPT_EVERY_STEP
        vec = isinstance(cost, AffineCost) and not cost.is_scalar
        if isinstance(cost, AffineCost):
            ck, a, b = (_lib.COST["affine"], 0.0, 0.0) if vec else (_lib.COST["affine"], float(cost.a), float(cost.b))
        else:
            ck, a, b = _lib.COST["explicit"], 0.0, 0.0
        self.handle.set_reverse_options(_lib.SA[sensealg], ck, a, b, flags, t)
        if vec or dgdp is not None:
            bc = lambda x, n: None if x is None else np.ascontiguousarray(np.broadcast_to(np.asarray(x, dtype=np.float64), (n,)))
            self.handle.set_cost_family(0, bc(cost.a, self.d) if vec else None, bc(cost.b, self.d) if vec else None,
                                        bc(getattr(dgdp, "c", None), self.P), bc(getattr(dgdp, "e", None), self.P))
        if t is not None:
            self.saveat = np.ascontiguousarray(t, dtype=np.float64)
            self.K = len(self.saveat)

    def step_counts(self):
        """(forward, reverse) accepted-step counts per member of an adaptive handle."""
        f, r = self._empty(self.N, dtype="i32", role="fwd_n"), self._empty(self.N, dtype="i32", role="rev_n")
        self.handle.step_counts(f, r)
        return f, r

    def noise(self):
        out = self._empty(self.S, self.m, self.N, role="noise")
        self.handle.get_noise(out)
        return out

    def close(self):
        self.handle.close()
