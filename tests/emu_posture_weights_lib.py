"""TEST INFRASTRUCTURE -- ctypes wrapper for tests/host_emu/emu_posture_weights.cpp: the pass loops of
bik_converge_weighted_ex / bik_track_weighted_ex (per-instance posture weights) compiled for the host (1 lane), next to the
unweighted and task-weighted loops that tests/emu_lib.py and tests/emu_weights_lib.py wrap."""

import ctypes as C
import os
import subprocess

import numpy as np

from tests.emu_lib import Emu, _as, _p, _vp

_HERE = os.path.join(os.path.dirname(os.path.abspath(__file__)), "host_emu")
_SO = os.path.join(_HERE, "_build", "libbikemu_posture_weights.so")
_lib = None


def lib():
    global _lib
    if _lib is None:
        src = os.path.join(_HERE, "emu_posture_weights.cpp")
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


class PostureWeightedEmu:
    """The posture-weighted pass loops on a problem of their own library.  Inputs as for Emu.converge / Emu.track, plus
    `weights` ([B, K] / [B, T, K]) and `posture_weights` ([B, P, nv] / [B, T, P, nv]) in q's dtype (None: the loop without
    them, which runs the unweighted K2).  posture_form: bik_inputs.posture_batched as given (2 and 3: target sequences)."""

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

    def k1_double(self, damping):
        """(without, with posture weights): whether K1 runs in fp64 for an fp32 caller."""
        out = np.zeros(2, np.int32)
        lib().emu_k1_double(self.h, C.c_double(damping), _p(out, C.c_int32))
        return bool(out[0]), bool(out[1])

    def converge(self, q, ftgt, ptgt, ctgt, posture_weights, dt, damping, max_iters, pos_threshold, ori_threshold, weights=None,
                 path=PATH_AUTO):
        """bik_converge_weighted_ex (..._ex64 for a float64 q).  Returns (q, iters, status)."""
        f64, q, ftgt, ptgt, ctgt, batched = self._loop_inputs(q, ftgt, ptgt, ctgt)
        B = q.shape[0]
        w, pw = _as(weights, q.dtype), _as(posture_weights, q.dtype)
        it = np.zeros(B, np.int32); st = np.zeros(B, np.int32)
        rc = lib().emu_converge_pw(self.h, f64, int(path), B, _vp(q), _vp(ftgt), _vp(ptgt), batched, _vp(ctgt), _vp(w), _vp(pw), C.c_double(dt),
                                   C.c_double(damping), int(max_iters), C.c_double(pos_threshold), C.c_double(ori_threshold),
                                   _p(it, C.c_int32), _p(st, C.c_int32))
        assert rc == 0, lib().emu_last_error()
        return q, it, st

    def track(self, q, ftgt, ptgt, ctgt, posture_weights, dt, damping, max_iters, pos_threshold, ori_threshold, lengths=None, weights=None,
              posture_form=None, path=PATH_AUTO):
        """bik_track_weighted_ex (..._ex64 for a float64 q).  Returns (q, q_traj, iters, status, passes) as Emu.track."""
        f64, q, ftgt, ptgt, ctgt, batched = self._loop_inputs(q, ftgt, ptgt, ctgt)
        if posture_form is not None:
            batched = int(posture_form)
        B, T = q.shape[0], (ftgt if ftgt is not None else ctgt).shape[1]
        w, pw = _as(weights, q.dtype), _as(posture_weights, q.dtype)
        q_traj = np.full((B, T, self.nq), np.nan, q.dtype)
        it = np.full((B, T), -1, np.int32); st = np.full((B, T), -1, np.int32); passes = np.zeros(1, np.int32)
        ln = _as(lengths, np.int32)
        rc = lib().emu_track_pw(self.h, f64, int(path), B, T, _vp(q), _vp(ftgt), _vp(ptgt), batched, _vp(ctgt), _vp(w), _vp(pw),
                                _p(ln, C.c_int32), C.c_double(dt), C.c_double(damping), int(max_iters), C.c_double(pos_threshold),
                                C.c_double(ori_threshold), _vp(q_traj), _p(it, C.c_int32), _p(st, C.c_int32), _p(passes, C.c_int32))
        assert rc == 0, lib().emu_last_error()
        return q, q_traj, it, st, int(passes[0])
