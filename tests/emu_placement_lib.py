"""TEST INFRASTRUCTURE -- ctypes wrapper for tests/host_emu/emu_placement.cpp: the step and the pass loops of bik_step_placed /
bik_converge_placed / bik_track_placed (per-instance frame placement) compiled for the host (1 lane), next to the loops they
fall back to without a placement (bik_step_coll, bik_converge_coll, bik_track_hold)."""

import ctypes as C
import copy
import math
import os
import subprocess

import numpy as np

from mink_b200._abi import TASK_FRAME, TASK_RELATIVE_FRAME
from mink_b200.flatten import Frame
from tests.emu_collision_lib import CollisionEmu
from tests.emu_lib import _as, _p, _vp

_HERE = os.path.join(os.path.dirname(os.path.abspath(__file__)), "host_emu")
_SO = os.path.join(_HERE, "_build", "libbikemu_placement.so")
_lib = None


def lib():
    global _lib
    if _lib is None:
        src = os.path.join(_HERE, "emu_placement.cpp")
        csrc = os.path.join(os.path.dirname(_HERE), "..", "mink_b200", "csrc")
        deps = [src] + [os.path.join(_HERE, f) for f in ("emu.cpp", "emu_bounds.cpp", "emu_collision.cpp", "emu_hold.cpp")] + \
               [os.path.join(csrc, f) for f in os.listdir(csrc) if f.endswith(".h")]
        if not os.path.exists(_SO) or any(os.path.getmtime(d) > os.path.getmtime(_SO) for d in deps):
            os.makedirs(os.path.dirname(_SO), exist_ok=True)
            subprocess.check_call(["g++", "-O2", "-std=c++17", "-shared", "-fPIC", "-Wno-unknown-pragmas", "-o", _SO, src])
        _lib = C.CDLL(_SO)
        _lib.emu_problem_create.restype = C.c_void_p
        _lib.emu_last_error.restype = C.c_char_p
    return _lib


def frame_tasks(spec):
    """The frame-like tasks of a spec (FRAME and RELATIVE_FRAME), in the order of the frame targets and placement rows."""
    return [t for t in spec.tasks if t.kind in (TASK_FRAME, TASK_RELATIVE_FRAME)]


def image_row(frame: Frame, dtype):
    """A frame's pose in its node as the problem image stores it (bik_build.h put_frame): the quaternion divided by its norm
    in double, then quaternion and position in `dtype`, wxyz_xyz."""
    q = [float(x) for x in frame.quat]
    n = math.sqrt(q[0] * q[0] + q[1] * q[1] + q[2] * q[2] + q[3] * q[3])
    return np.array([x / n for x in q] + [float(x) for x in frame.pos]).astype(dtype)


def own_placement(spec, B, dtype):
    """[B, F, 7] rows that hold the problem's own placement of every frame task."""
    rows = np.stack([image_row(t.frame, dtype) for t in frame_tasks(spec)])
    return np.ascontiguousarray(np.broadcast_to(rows, (B,) + rows.shape))


def placed_spec(spec, rows):
    """The spec with frame task f's frame at rows[f] (wxyz_xyz) in its node: the problem a placement stands for."""
    out = copy.deepcopy(spec)
    for t, r in zip(frame_tasks(out), rows):
        r = np.asarray(r, dtype=np.float64)
        t.frame = Frame(t.frame.node, r[4:].copy(), r[:4].copy())
    return out


class PlacementEmu(CollisionEmu):
    """The placed step and pass loops on a problem of this library.  Inputs as for CollisionEmu, plus placement [B, F, 7] in
    q's dtype (None: the loop without a placement) and, for track, hold [B, T, F + C + P] (or None)."""

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

    def step(self, q, ftgt, ptgt, ctgt, placement, dt, damping, nsteps=1, coll=None, f32k1=False):
        """bik_step_placed (bik_step_coll for placement None), integrating q.  Returns (q, dq, status)."""
        f64, q, ftgt, ptgt, ctgt, batched = self._loop_inputs(q, ftgt, ptgt, ctgt)
        B = q.shape[0]
        en, dmin, ddet = self._coll(coll, q.dtype)
        pl = _as(placement, q.dtype)
        dq = np.zeros((B, self.nv), q.dtype); st = np.zeros(B, np.int32)
        rc = lib().emu_step_placed(self.h, f64, int(bool(f32k1)), B, _vp(q), _vp(ftgt), _vp(ptgt), batched, _vp(ctgt), _vp(en), _vp(dmin),
                                   _vp(ddet), _vp(pl), C.c_double(dt), C.c_double(damping), int(nsteps), 1, _vp(dq), _p(st, C.c_int32))
        assert rc == 0, lib().emu_last_error()
        return q, dq, st

    def converge(self, q, ftgt, ptgt, ctgt, placement, dt, damping, max_iters, pos_threshold, ori_threshold, coll=None, f32k1=False):
        """bik_converge_placed (bik_converge_coll for placement None).  Returns (q, iters, status)."""
        f64, q, ftgt, ptgt, ctgt, batched = self._loop_inputs(q, ftgt, ptgt, ctgt)
        B = q.shape[0]
        en, dmin, ddet = self._coll(coll, q.dtype)
        pl = _as(placement, q.dtype)
        it = np.zeros(B, np.int32); st = np.zeros(B, np.int32)
        rc = lib().emu_loop_placed(self.h, f64, int(bool(f32k1)), 0, B, 1, _vp(q), _vp(ftgt), _vp(ptgt), batched, _vp(ctgt), _vp(en), _vp(dmin),
                                   _vp(ddet), None, _vp(pl), None, C.c_double(dt), C.c_double(damping), int(max_iters),
                                   C.c_double(pos_threshold), C.c_double(ori_threshold), None, _p(it, C.c_int32), _p(st, C.c_int32), None)
        assert rc == 0, lib().emu_last_error()
        return q, it, st

    def track(self, q, ftgt, ptgt, ctgt, placement, dt, damping, max_iters, pos_threshold, ori_threshold, hold=None, coll=None,
              lengths=None, f32k1=False):
        """bik_track_placed (bik_track_hold for placement None).  Returns (q, q_traj, iters, status, passes)."""
        f64, q, ftgt, ptgt, ctgt, batched = self._loop_inputs(q, ftgt, ptgt, ctgt)
        B, T = q.shape[0], (ftgt if ftgt is not None else ctgt).shape[1]
        en, dmin, ddet = self._coll(coll, q.dtype)
        pl = _as(placement, q.dtype)
        hd = None if hold is None else np.ascontiguousarray(np.asarray(hold) != 0, dtype=np.uint8)
        q_traj = np.full((B, T, self.nq), np.nan, q.dtype)
        it = np.full((B, T), -1, np.int32); st = np.full((B, T), -1, np.int32); passes = np.zeros(1, np.int32)
        ln = _as(lengths, np.int32)
        rc = lib().emu_loop_placed(self.h, f64, int(bool(f32k1)), 1, B, T, _vp(q), _vp(ftgt), _vp(ptgt), batched, _vp(ctgt), _vp(en),
                                   _vp(dmin), _vp(ddet), _vp(hd), _vp(pl), _p(ln, C.c_int32), C.c_double(dt), C.c_double(damping),
                                   int(max_iters), C.c_double(pos_threshold), C.c_double(ori_threshold), _vp(q_traj), _p(it, C.c_int32),
                                   _p(st, C.c_int32), _p(passes, C.c_int32))
        assert rc == 0, lib().emu_last_error()
        return q, q_traj, it, st, int(passes[0])
