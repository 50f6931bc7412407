"""TEST INFRASTRUCTURE -- ctypes wrapper for tests/host_emu/emu_bounds.cpp: the pass loops of bik_converge_bounded /
bik_track_bounded (per-instance bounds) compiled for the host (1 lane), next to the loops that tests/emu_lib.py,
tests/emu_weights_lib.py and tests/emu_posture_weights_lib.py wrap."""

import ctypes as C
import os
import subprocess

import numpy as np

from tests.emu_lib import Emu, _as, _p, _vp

_HERE = os.path.join(os.path.dirname(os.path.abspath(__file__)), "host_emu")
_SO = os.path.join(_HERE, "_build", "libbikemu_bounds.so")
_lib = None


def lib():
    global _lib
    if _lib is None:
        src = os.path.join(_HERE, "emu_bounds.cpp")
        csrc = os.path.join(os.path.dirname(_HERE), "..", "mink_b200", "csrc")
        deps = [src, os.path.join(_HERE, "emu.cpp")] + [os.path.join(csrc, f) for f in os.listdir(csrc) if f.endswith(".h")]
        if not os.path.exists(_SO) or any(os.path.getmtime(d) > os.path.getmtime(_SO) for d in deps):
            os.makedirs(os.path.dirname(_SO), exist_ok=True)
            subprocess.check_call(["g++", "-O2", "-std=c++17", "-shared", "-fPIC", "-Wno-unknown-pragmas", "-o", _SO, src])
        _lib = C.CDLL(_SO)
        _lib.emu_problem_create.restype = C.c_void_p
        _lib.emu_last_error.restype = C.c_char_p
    return _lib


# K2 path: the device's choice, or the general path (what BIK_K2_PATH=dense selects on the device)
PATH_AUTO, PATH_GENERAL = 0, 1


class BoundedEmu:
    """The bounded pass loops on a problem of their own library.  Inputs as for Emu.converge / Emu.track, plus `bounds`
    (lower, upper, vmax), each [B, nv] in q's dtype or None (all None: the ..._weighted_ex loop), and optionally `weights`
    ([B, K] / [B, T, K]) and `posture_weights` ([B, P, nv] / [B, T, P, nv]).  posture_form: bik_inputs.posture_batched as
    given (2 and 3: target sequences)."""

    def __init__(self, blob: bytes, spec, nq, nv):
        self.spec, self.nq, self.nv = spec, nq, nv
        t, nt, l, nl, self._keep = spec.to_c()
        h = lib().emu_problem_create(blob, len(blob), t, nt, l, nl)
        if not h:
            raise RuntimeError(lib().emu_last_error().decode())
        self.h = C.c_void_p(h)

    def __del__(self):
        if getattr(self, "h", None):
            lib().emu_problem_destroy(self.h)

    _loop_inputs = Emu._loop_inputs

    @staticmethod
    def _bounds(bounds, dtype):
        lo, up, vm = bounds if bounds is not None else (None, None, None)
        return _as(lo, dtype), _as(up, dtype), _as(vm, dtype)

    def converge(self, q, ftgt, ptgt, ctgt, bounds, dt, damping, max_iters, pos_threshold, ori_threshold, weights=None,
                 posture_weights=None, path=PATH_AUTO):
        """bik_converge_bounded (..._bounded64 for a float64 q).  Returns (q, iters, status)."""
        f64, q, ftgt, ptgt, ctgt, batched = self._loop_inputs(q, ftgt, ptgt, ctgt)
        B = q.shape[0]
        w, pw = _as(weights, q.dtype), _as(posture_weights, q.dtype)
        lo, up, vm = self._bounds(bounds, q.dtype)
        it = np.zeros(B, np.int32); st = np.zeros(B, np.int32)
        rc = lib().emu_converge_bd(self.h, f64, int(path), B, _vp(q), _vp(ftgt), _vp(ptgt), batched, _vp(ctgt), _vp(w), _vp(pw), _vp(lo),
                                   _vp(up), _vp(vm), C.c_double(dt), C.c_double(damping), int(max_iters), C.c_double(pos_threshold),
                                   C.c_double(ori_threshold), _p(it, C.c_int32), _p(st, C.c_int32))
        assert rc == 0, lib().emu_last_error()
        return q, it, st

    def track(self, q, ftgt, ptgt, ctgt, bounds, dt, damping, max_iters, pos_threshold, ori_threshold, lengths=None, weights=None,
              posture_weights=None, posture_form=None, path=PATH_AUTO):
        """bik_track_bounded (..._bounded64 for a float64 q).  Returns (q, q_traj, iters, status, passes) as Emu.track."""
        f64, q, ftgt, ptgt, ctgt, batched = self._loop_inputs(q, ftgt, ptgt, ctgt)
        if posture_form is not None:
            batched = int(posture_form)
        B, T = q.shape[0], (ftgt if ftgt is not None else ctgt).shape[1]
        w, pw = _as(weights, q.dtype), _as(posture_weights, q.dtype)
        lo, up, vm = self._bounds(bounds, q.dtype)
        q_traj = np.full((B, T, self.nq), np.nan, q.dtype)
        it = np.full((B, T), -1, np.int32); st = np.full((B, T), -1, np.int32); passes = np.zeros(1, np.int32)
        ln = _as(lengths, np.int32)
        rc = lib().emu_track_bd(self.h, f64, int(path), B, T, _vp(q), _vp(ftgt), _vp(ptgt), batched, _vp(ctgt), _vp(w), _vp(pw), _vp(lo),
                                _vp(up), _vp(vm), _p(ln, C.c_int32), C.c_double(dt), C.c_double(damping), int(max_iters),
                                C.c_double(pos_threshold), C.c_double(ori_threshold), _vp(q_traj), _p(it, C.c_int32), _p(st, C.c_int32),
                                _p(passes, C.c_int32))
        assert rc == 0, lib().emu_last_error()
        return q, q_traj, it, st, int(passes[0])
