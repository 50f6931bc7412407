"""TEST INFRASTRUCTURE -- ctypes wrapper for tests/host_emu/emu_hold.cpp: the pass loop of bik_track_hold (held targets)
compiled for the host (1 lane), and the reference values a held task captures, from the emulated bik_fk."""

import ctypes as C
import os
import subprocess

import numpy as np

from mink_b200._abi import TASK_COM, TASK_FRAME, TASK_POSTURE, TASK_RELATIVE_FRAME, c_frames
from tests.emu_collision_lib import CollisionEmu
from tests.emu_lib import _as, _p, _vp

_HERE = os.path.join(os.path.dirname(os.path.abspath(__file__)), "host_emu")
_SO = os.path.join(_HERE, "_build", "libbikemu_hold.so")
_lib = None


def lib():
    global _lib
    if _lib is None:
        src = os.path.join(_HERE, "emu_hold.cpp")
        csrc = os.path.join(os.path.dirname(_HERE), "..", "mink_b200", "csrc")
        deps = [src] + [os.path.join(_HERE, f) for f in ("emu.cpp", "emu_bounds.cpp", "emu_collision.cpp")] + \
               [os.path.join(csrc, f) for f in os.listdir(csrc) if f.endswith(".h")]
        if not os.path.exists(_SO) or any(os.path.getmtime(d) > os.path.getmtime(_SO) for d in deps):
            os.makedirs(os.path.dirname(_SO), exist_ok=True)
            subprocess.check_call(["g++", "-O2", "-std=c++17", "-shared", "-fPIC", "-Wno-unknown-pragmas", "-o", _SO, src])
        _lib = C.CDLL(_SO)
        _lib.emu_problem_create.restype = C.c_void_p
        _lib.emu_last_error.restype = C.c_char_p
    return _lib


class HoldEmu(CollisionEmu):
    """The bik_track_hold loop, next to the bik_converge_coll / bik_track_coll loops (CollisionEmu) and the emulated bik_fk,
    all on one problem of this library."""

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

    def converge(self, q, ftgt, ptgt, ctgt, dt, damping, max_iters, pos_threshold, ori_threshold, f32k1=False):
        """bik_converge_coll without collision arguments, i.e. bik_converge (..._64 for a float64 q).  Returns (q, iters, status)."""
        f64, q, ftgt, ptgt, ctgt, batched = self._loop_inputs(q, ftgt, ptgt, ctgt)
        B = q.shape[0]
        it = np.zeros(B, np.int32); st = np.zeros(B, np.int32)
        rc = lib().emu_converge_coll(self.h, f64, int(bool(f32k1)), B, _vp(q), _vp(ftgt), _vp(ptgt), batched, _vp(ctgt), None, None, None,
                                     None, C.c_double(dt), C.c_double(damping), int(max_iters), C.c_double(pos_threshold),
                                     C.c_double(ori_threshold), _p(it, C.c_int32), _p(st, C.c_int32))
        assert rc == 0, lib().emu_last_error()
        return q, it, st

    def fk(self, q, frames, f64):
        """The emulated bik_fk (bik_fk64): (poses [B, nframes, 7], com [B, 3])."""
        t = np.float64 if f64 else np.float32
        q = _as(q, t); B = q.shape[0]
        poses = np.zeros((B, len(frames), 7), t); com = np.zeros((B, 3), t)
        assert lib().emu_fk(self.h, B, int(f64), _vp(q), c_frames(frames), len(frames), _vp(poses), _vp(com), None) == 0
        return poses, com

    def track_hold(self, q, ftgt, ptgt, ctgt, hold, dt, damping, max_iters, pos_threshold, ori_threshold, coll=None, lengths=None,
                   f32k1=False):
        """bik_track_hold (..._hold64 for a float64 q); hold [B, T, F + C + P] or None (the bik_track_coll loop).  Returns
        (q, q_traj, iters, status, passes) as Emu.track."""
        f64, q, ftgt, ptgt, ctgt, batched = self._loop_inputs(q, ftgt, ptgt, ctgt)
        B, T = q.shape[0], (ftgt if ftgt is not None else ctgt).shape[1]
        en, dmin, ddet = self._coll(coll, q.dtype)
        hd = None if hold is None else np.ascontiguousarray(np.asarray(hold) != 0, dtype=np.uint8)
        q_traj = np.full((B, T, self.nq), np.nan, q.dtype)
        it = np.full((B, T), -1, np.int32); st = np.full((B, T), -1, np.int32); passes = np.zeros(1, np.int32)
        ln = _as(lengths, np.int32)
        rc = lib().emu_track_hold(self.h, f64, int(bool(f32k1)), B, T, _vp(q), _vp(ftgt), _vp(ptgt), batched, _vp(ctgt), None, _vp(en),
                                  _vp(dmin), _vp(ddet), _vp(hd), _p(ln, C.c_int32), C.c_double(dt), C.c_double(damping), int(max_iters),
                                  C.c_double(pos_threshold), C.c_double(ori_threshold), _vp(q_traj), _p(it, C.c_int32), _p(st, C.c_int32),
                                  _p(passes, C.c_int32))
        assert rc == 0, lib().emu_last_error()
        return q, q_traj, it, st, int(passes[0])

    def capture(self, q, f64):
        """What each held task captures at q [B, nq], from the emulated bik_fk in fp64 (f64) or fp32, in q's dtype: a list
        over the F frame-like tasks, C CoM tasks and P posture-type tasks, in hold-column order, of [B, 7] / [B, 3] / [B, nq]."""
        tasks = self.spec.tasks
        fr = [t for t in tasks if t.kind in (TASK_FRAME, TASK_RELATIVE_FRAME)]
        roots = [t.root for t in fr if t.kind == TASK_RELATIVE_FRAME]
        t = np.float64 if f64 else np.float32
        poses, com = self.fk(np.asarray(q, t), [x.frame for x in fr] + roots, f64=f64)
        out, r = [], len(fr)
        for i, x in enumerate(fr):
            p = poses[:, i]
            if x.kind == TASK_RELATIVE_FRAME:
                root, frame, rel = np.ascontiguousarray(poses[:, r]), np.ascontiguousarray(p), np.zeros_like(p)
                lib().emu_relative_pose(int(f64), p.shape[0], _vp(root), _vp(frame), _vp(rel))
                p, r = rel, r + 1
            out.append(p)
        out += [com for x in tasks if x.kind == TASK_COM]
        out += [np.asarray(q) for x in tasks if x.kind == TASK_POSTURE]
        return [np.asarray(v).astype(np.asarray(q).dtype) for v in out]
