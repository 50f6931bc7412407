"""TEST INFRASTRUCTURE -- ctypes wrapper for tests/host_emu/track64_emu.cpp: the pass loops of bik_converge64 and bik_track64
with the kernel headers compiled for the host (one lane per instance, fp64 buffers, collision rows included)."""

import ctypes as C
import os
import subprocess

import numpy as np

_HERE = os.path.join(os.path.dirname(os.path.abspath(__file__)), "host_emu")
_SO = os.path.join(_HERE, "_build", "libbiktrack64emu.so")
_lib = None


def lib():
    global _lib
    if _lib is None:
        src = os.path.join(_HERE, "track64_emu.cpp")
        csrc = os.path.join(os.path.dirname(_HERE), "..", "mink_b200", "csrc")
        deps = [src] + [os.path.join(csrc, f) for f in os.listdir(csrc) if f.endswith(".h")]
        if not os.path.exists(_SO) or any(os.path.getmtime(d) > os.path.getmtime(_SO) for d in deps):
            os.makedirs(os.path.dirname(_SO), exist_ok=True)
            subprocess.check_call(["g++", "-O2", "-std=c++17", "-shared", "-fPIC", "-Wno-unknown-pragmas", "-o", _SO, src])
        _lib = C.CDLL(_SO)
        _lib.track64_emu_problem_create.restype = C.c_void_p
        _lib.track64_emu_problem_destroy.argtypes = [C.c_void_p]
        _lib.track64_emu_last_error.restype = C.c_char_p
    return _lib


def _p(a, t=C.c_double):
    return None if a is None else a.ctypes.data_as(C.POINTER(t))


def _as(a, dt=np.float64):
    return None if a is None else np.ascontiguousarray(a, dtype=dt)


class Track64Emu:
    def __init__(self, blob: bytes, spec, nq, nv):
        self.spec, self.nq, self.nv = spec, nq, nv
        t, nt, l, nl, self._keep = spec.to_c()
        h = lib().track64_emu_problem_create(blob, len(blob), t, nt, l, nl)
        if not h:
            raise RuntimeError(lib().track64_emu_last_error().decode())
        self.h = C.c_void_p(h)

    def __del__(self):
        h, self.h = getattr(self, "h", None), None
        if h:
            lib().track64_emu_problem_destroy(h)

    def _inputs(self, q, ftgt, ptgt, ctgt):
        q = _as(q).copy()
        ftgt, ptgt, ctgt = _as(ftgt), _as(ptgt), _as(ctgt)
        B = q.shape[0]
        batched = int(ptgt is not None and ptgt.size == B * self.spec.nposture * self.nq and B > 1)
        return q, ftgt, ptgt, ctgt, batched

    def _check(self, rc):
        assert rc == 0, lib().track64_emu_last_error().decode()

    def converge(self, q, ftgt, ptgt, ctgt, dt, damping, max_iters, pos_threshold, ori_threshold):
        """The pass loop of bik_converge64.  Returns (q, iters, status)."""
        q, ftgt, ptgt, ctgt, batched = self._inputs(q, ftgt, ptgt, ctgt)
        B = q.shape[0]
        it = np.zeros(B, np.int32); st = np.zeros(B, np.int32)
        self._check(lib().track64_emu_converge(self.h, B, _p(q), _p(ftgt), _p(ptgt), batched, _p(ctgt), C.c_double(dt),
                                               C.c_double(damping), int(max_iters), C.c_double(pos_threshold),
                                               C.c_double(ori_threshold), _p(it, C.c_int32), _p(st, C.c_int32)))
        return q, it, st

    def track(self, q, ftgt, ptgt, ctgt, dt, damping, max_iters, pos_threshold, ori_threshold, lengths=None):
        """The pass loop of bik_track64: ftgt [B,T,F,7], ctgt [B,T,C,3].  Returns (q, q_traj, iters, status, passes); rows
        past an instance's length hold NaN / -1 / -1."""
        q, ftgt, ptgt, ctgt, batched = self._inputs(q, ftgt, ptgt, ctgt)
        B, T = q.shape[0], (ftgt if ftgt is not None else ctgt).shape[1]
        q_traj = np.full((B, T, self.nq), np.nan)
        it = np.full((B, T), -1, np.int32); st = np.full((B, T), -1, np.int32); passes = np.zeros(1, np.int32)
        ln = _as(lengths, np.int32)
        self._check(lib().track64_emu_track(self.h, B, T, _p(q), _p(ftgt), _p(ptgt), batched, _p(ctgt), _p(ln, C.c_int32),
                                            C.c_double(dt), C.c_double(damping), int(max_iters), C.c_double(pos_threshold),
                                            C.c_double(ori_threshold), _p(q_traj), _p(it, C.c_int32), _p(st, C.c_int32),
                                            _p(passes, C.c_int32)))
        return q, q_traj, it, st, int(passes[0])
