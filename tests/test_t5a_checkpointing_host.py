"""CPU-side plumbing of the checkpointed save intervals on the adaptive Tsit5 path (B200ADJ_FLAG_CHECKPOINT_SAVES) and of
b200adj_device_bytes: the flag bit and its create-time class, the host objects that carry it, the exported entry point."""
import ctypes as C
import os
import re

import numpy as np
import pytest

import scimlsensitivity_jl_b200 as b
from scimlsensitivity_jl_b200 import _lib, concrete_solve

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
HDR = open(os.path.join(ROOT, "include", "b200adj.h")).read()


def test_flag_bit_matches_the_header_and_is_a_create_flag():
    m = re.search(r"#define B200ADJ_FLAG_CHECKPOINT_SAVES\s+(\d+)u", HDR)
    assert m and int(m.group(1)) == _lib.FLAG_CHECKPOINT_SAVES
    create = re.search(r"#define B200ADJ_CREATE_FLAGS \(([^)]*)\)", HDR, re.S).group(1)
    assert "B200ADJ_FLAG_CHECKPOINT_SAVES" in create
    others = [_lib.FLAG_NO_START, _lib.FLAG_NO_CHECKPOINTING, _lib.FLAG_CKPT_EVERY_STEP, _lib.FLAG_STORED_NOISE, _lib.FLAG_TRACE,
              _lib.FLAG_NO_ROTATE, _lib.FLAG_DENSE_FORWARD, _lib.FLAG_NCCL_ALLREDUCE]
    assert all(_lib.FLAG_CHECKPOINT_SAVES & f == 0 for f in others)


def test_device_bytes_is_declared_exported_and_bound():
    assert re.search(r"int32_t b200adj_device_bytes\(void\* handle, int64_t\* bytes\);", HDR)
    assert "b200adj_device_bytes" in _lib.EXPORTS
    lib = _lib.load()
    fn = lib.b200adj_device_bytes
    assert fn.restype == C.c_int32 and fn.argtypes == [C.c_void_p, C.POINTER(C.c_int64)]
    n = C.c_int64(7)
    assert fn(None, C.byref(n)) == -1 and n.value == 7          # null handle: B200ADJ_ERR_INVALID, nothing written


def test_b200adjoint_carries_the_mode():
    assert b.B200Adjoint(b.GaussAdjoint()).checkpoint_saves is False
    sa = b.B200Adjoint(b.GaussAdjoint(), checkpoint_saves=True)
    assert sa.checkpoint_saves is True and isinstance(sa.inner, b.GaussAdjoint)
    # the plain reference keyword keeps its meaning: no B200 flag follows from it
    assert b.InterpolatingAdjoint(checkpointing=True).checkpointing is True
    assert not hasattr(b.InterpolatingAdjoint(checkpointing=True), "checkpoint_saves")


def test_device_ensemble_sets_the_flag_and_the_cache_key_holds_it(monkeypatch):
    seen = []

    class FakeHandle:
        def __init__(self, cfg, saveat):
            seen.append(int(cfg.flags))

        def set_stream(self, ptr):
            pass

    monkeypatch.setattr(_lib, "Handle", FakeHandle)
    for ck in (False, True):
        b.DeviceEnsemble("lv", "gauss", "tsit5_adaptive", 4, np.linspace(0.0, 1.0, 3), (0.0, 1.0), 0.0, checkpoint_saves=ck)
    assert seen[0] & _lib.FLAG_CHECKPOINT_SAVES == 0 and seen[1] & _lib.FLAG_CHECKPOINT_SAVES
    # solve() keys its handle cache on the mode: the two sensealgs must not share a handle
    src = open(concrete_solve.__file__).read()
    key = src[src.index("    key = ("):src.index("    eng = _HANDLE_CACHE.get(key)")]
    assert "ckpt_saves" in key and "checkpoint_saves=ckpt_saves" in src
