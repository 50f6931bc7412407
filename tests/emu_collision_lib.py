"""TEST INFRASTRUCTURE -- ctypes wrapper for tests/host_emu/emu_collision.cpp: the pass loops of bik_converge_coll /
bik_track_coll (per-instance collision pairs and distances) compiled for the host (1 lane), and one K1 of a step with them,
next to the loops that tests/emu_lib.py and tests/emu_bounds_lib.py wrap."""

import ctypes as C
import os
import subprocess

import numpy as np

from tests.emu_lib import Emu, _as, _p, _vp

_HERE = os.path.join(os.path.dirname(os.path.abspath(__file__)), "host_emu")
_SO = os.path.join(_HERE, "_build", "libbikemu_collision.so")
_lib = None


def lib():
    global _lib
    if _lib is None:
        src = os.path.join(_HERE, "emu_collision.cpp")
        csrc = os.path.join(os.path.dirname(_HERE), "..", "mink_b200", "csrc")
        deps = [src, os.path.join(_HERE, "emu.cpp"), os.path.join(_HERE, "emu_bounds.cpp")] + \
               [os.path.join(csrc, f) for f in os.listdir(csrc) if f.endswith(".h")]
        if not os.path.exists(_SO) or any(os.path.getmtime(d) > os.path.getmtime(_SO) for d in deps):
            os.makedirs(os.path.dirname(_SO), exist_ok=True)
            subprocess.check_call(["g++", "-O2", "-std=c++17", "-shared", "-fPIC", "-Wno-unknown-pragmas", "-o", _SO, src])
        _lib = C.CDLL(_SO)
        _lib.emu_problem_create.restype = C.c_void_p
        _lib.emu_last_error.restype = C.c_char_p
    return _lib


class CollisionEmu:
    """The collision pass loops on a problem of their own library.  Inputs as for Emu.converge / Emu.track, plus `coll`
    (enabled, minimum_distance, detection_distance): enabled [B, npairs] (track: [B, T, npairs]) bools, the distances [B]
    (track: [B, T]) in q's dtype, each None (all None: the ..._bounded loop without bounds).  f32k1: K1 in fp32 for fp32
    callers (BIK_K1_PRECISION=f32)."""

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
    def _coll(coll, dtype):
        en, dmin, ddet = coll if coll is not None else (None, None, None)
        en = None if en is None else np.ascontiguousarray(np.asarray(en) != 0, dtype=np.uint8)
        return en, _as(dmin, dtype), _as(ddet, dtype)

    def converge(self, q, ftgt, ptgt, ctgt, coll, dt, damping, max_iters, pos_threshold, ori_threshold, posture_weights=None, f32k1=False):
        """bik_converge_coll (..._coll64 for a float64 q).  Returns (q, iters, status)."""
        f64, q, ftgt, ptgt, ctgt, batched = self._loop_inputs(q, ftgt, ptgt, ctgt)
        B = q.shape[0]
        pw = _as(posture_weights, q.dtype)
        en, dmin, ddet = self._coll(coll, q.dtype)
        it = np.zeros(B, np.int32); st = np.zeros(B, np.int32)
        rc = lib().emu_converge_coll(self.h, f64, int(bool(f32k1)), B, _vp(q), _vp(ftgt), _vp(ptgt), batched, _vp(ctgt), _vp(pw), _vp(en),
                                     _vp(dmin), _vp(ddet), C.c_double(dt), C.c_double(damping), int(max_iters), C.c_double(pos_threshold),
                                     C.c_double(ori_threshold), _p(it, C.c_int32), _p(st, C.c_int32))
        assert rc == 0, lib().emu_last_error()
        return q, it, st

    def track(self, q, ftgt, ptgt, ctgt, coll, dt, damping, max_iters, pos_threshold, ori_threshold, lengths=None, posture_weights=None,
              f32k1=False):
        """bik_track_coll (..._coll64 for a float64 q).  Returns (q, q_traj, iters, status, passes) as Emu.track."""
        f64, q, ftgt, ptgt, ctgt, batched = self._loop_inputs(q, ftgt, ptgt, ctgt)
        B, T = q.shape[0], (ftgt if ftgt is not None else ctgt).shape[1]
        pw = _as(posture_weights, q.dtype)
        en, dmin, ddet = self._coll(coll, q.dtype)
        q_traj = np.full((B, T, self.nq), np.nan, q.dtype)
        it = np.full((B, T), -1, np.int32); st = np.full((B, T), -1, np.int32); passes = np.zeros(1, np.int32)
        ln = _as(lengths, np.int32)
        rc = lib().emu_track_coll(self.h, f64, int(bool(f32k1)), B, T, _vp(q), _vp(ftgt), _vp(ptgt), batched, _vp(ctgt), _vp(pw), _vp(en),
                                  _vp(dmin), _vp(ddet), _p(ln, C.c_int32), C.c_double(dt), C.c_double(damping), int(max_iters),
                                  C.c_double(pos_threshold), C.c_double(ori_threshold), _vp(q_traj), _p(it, C.c_int32), _p(st, C.c_int32),
                                  _p(passes, C.c_int32))
        assert rc == 0, lib().emu_last_error()
        return q, q_traj, it, st, int(passes[0])

    def k1(self, q, ftgt, ptgt, ctgt, coll, dt):
        """One K1 of a step in fp64 (the precision collision problems take) with collision arguments: (Gc [B, npairs, nv],
        hc [B, npairs], status [B])."""
        f64, q, ftgt, ptgt, ctgt, batched = self._loop_inputs(q, ftgt, ptgt, ctgt)
        B, npairs = q.shape[0], self.spec.npairs
        en, dmin, ddet = self._coll(coll, q.dtype)
        hdr = np.zeros(32, np.int32)
        lib().emu_header(self.h, _p(hdr, C.c_int32))
        pk = np.zeros((B, max(int(hdr[8]), 4)))   # pk_stride
        Gc = np.full((B, max(npairs, 1), self.nv), np.nan)
        hc = np.full((B, max(npairs, 1)), np.nan)
        st = np.zeros(B, np.int32)
        rc = lib().emu_k1_coll(self.h, B, 1 if f64 else 2, _vp(q), _vp(ftgt), _vp(ptgt), batched, _vp(ctgt), C.c_double(dt), _vp(en), _vp(dmin),
                               _vp(ddet), _vp(pk), _vp(Gc), _vp(hc), _p(st, C.c_int32))
        assert rc == 0, lib().emu_last_error()
        return Gc, hc, st
