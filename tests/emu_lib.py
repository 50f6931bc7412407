"""TEST INFRASTRUCTURE -- ctypes wrapper for tests/host_emu (kernel headers compiled for the host, 1 lane)."""

import ctypes as C
import os
import subprocess

import numpy as np

from mink_b200._abi import c_frames

_HERE = os.path.join(os.path.dirname(os.path.abspath(__file__)), "host_emu")
_SO = os.path.join(_HERE, "_build", "libbikemu.so")
_lib = None


def lib():
    global _lib
    if _lib is None:
        src = os.path.join(_HERE, "emu.cpp")
        csrc = os.path.join(os.path.dirname(_HERE), "..", "mink_b200", "csrc")
        deps = [src] + [os.path.join(csrc, f) for f in os.listdir(csrc) if f.endswith(".h")]
        if not os.path.exists(_SO) or any(os.path.getmtime(d) > os.path.getmtime(_SO) for d in deps):
            os.makedirs(os.path.dirname(_SO), exist_ok=True)
            subprocess.check_call(["g++", "-O2", "-std=c++17", "-shared", "-fPIC", "-Wno-unknown-pragmas", "-o", _SO, src])
        _lib = C.CDLL(_SO)
        _lib.emu_problem_create.restype = C.c_void_p
        _lib.emu_last_error.restype = C.c_char_p
    return _lib


def _vp(a):
    return None if a is None else C.c_void_p(a.ctypes.data)


def _p(a, t=C.c_float):
    return None if a is None else a.ctypes.data_as(C.POINTER(t))


def _as(a, dt):
    return None if a is None else np.ascontiguousarray(a, dtype=dt)


class Emu:
    def __init__(self, blob: bytes, spec, nq, nv):
        self.spec, self.nq, self.nv = spec, nq, nv
        t, nt, l, nl, self._keep = spec.to_c()
        self.h = lib().emu_problem_create(blob, len(blob), t, nt, l, nl)
        if not self.h:
            raise RuntimeError(lib().emu_last_error().decode())
        self.h = C.c_void_p(self.h)

    def header(self):
        """Fields of the problem image the CPU tests pin."""
        out = np.zeros(16, np.int32)
        lib().emu_header(self.h, _p(out, C.c_int32))
        names = ("nv", "nu", "nfree", "nnode", "nneeded", "nslots", "G", "nsteps", "pk_stride", "words32", "words")
        return dict(zip(names, (int(v) for v in out)))

    def set_knobs(self, sweeps: int):
        lib().emu_set_knobs(self.h, int(sweeps))

    def fk_jac(self, q, ftgt=None, ptgt=None, ctgt=None, dt=1e-2, prec="f32", packed=False, check=False):
        """K1.  prec: "f32" (fp32 kernel, fp32 buffers), "f64" (fp64 kernel, fp64 buffers), "mixed" (fp64 kernel on fp32
        inputs, fp64 outputs).  packed=True returns (pk, Gc, hc) instead of (J, e, ep, Gc, hc); check=True appends status."""
        s = self.spec
        tin = np.float64 if prec == "f64" else np.float32
        tout = np.float32 if prec == "f32" else np.float64
        mode = {"f32": 0, "f64": 1, "mixed": 2}[prec]
        q = _as(q, tin); B = q.shape[0]
        ftgt, ptgt, ctgt = _as(ftgt, tin), _as(ptgt, tin), _as(ctgt, tin)
        Gc = np.zeros((B, max(s.npairs, 1), self.nv), tout); hc = np.zeros((B, max(s.npairs, 1)), tout)
        batched = int(ptgt is not None and ptgt.size == B * s.nposture * self.nq and B > 1)
        st = np.zeros(B, np.int32) if check else None
        if packed:
            pk = np.full((B, self.header()["pk_stride"]), np.nan, tout)
            lib().emu_fk_jac(self.h, B, mode, _vp(q), _vp(ftgt), _vp(ptgt), batched, _vp(ctgt), C.c_double(dt), None, None, None,
                             _vp(Gc), _vp(hc), _vp(pk), _p(st, C.c_int32))
            out = (pk, Gc[:, :s.npairs], hc[:, :s.npairs])
        else:
            J = np.zeros((B, s.nrows, self.nv), tout); e = np.zeros((B, max(s.nrows, 1)), tout)
            ep = np.zeros((B, max(s.nposture, 1), self.nv), tout)
            lib().emu_fk_jac(self.h, B, mode, _vp(q), _vp(ftgt), _vp(ptgt), batched, _vp(ctgt), C.c_double(dt), _vp(J), _vp(e), _vp(ep),
                             _vp(Gc), _vp(hc), None, _p(st, C.c_int32))
            out = (J, e[:, :s.nrows], ep[:, :s.nposture], Gc[:, :s.npairs], hc[:, :s.npairs])
        return out + (st,) if check else out

    def solve(self, q, J, e, ep, Gc, hc, dt, damping, use_double=True, want_objective=False, io64=False, pk=None, ptgt=None,
              integrate=False, warm=None, skip=None, dq_inout=None):
        """K2, fp64 solve.  use_double: True/1 general path, 3 small-group, 8 small-group with 64-bit masks (packed fp32
        rows with fp32 I/O take the small-group step instantiation).  Task rows dense (J, e, ep) or packed (pk; then the
        posture error comes from q and ptgt).  Returns (dq, status, iters, H, c, lo, hi) (+ q after integration when
        integrate=True)."""
        s = self.spec
        path = int(use_double)
        tio = np.float64 if io64 else np.float32
        q = _as(q, tio).copy(); B = q.shape[0]
        pad = lambda a: None if a is None else np.ascontiguousarray(a if a.shape[1] else np.zeros((B, 1) + a.shape[2:], a.dtype))
        dq = dq_inout if dq_inout is not None else np.zeros((B, self.nv), tio)
        assert dq.dtype == tio and dq.flags.c_contiguous
        st = np.zeros(B, np.int32); it = np.zeros(B, np.int32)
        H = np.zeros((B, self.nv, self.nv)) if want_objective else None
        c = np.zeros((B, self.nv)) if want_objective else None
        lo = np.zeros((B, self.nv), tio); hi = np.zeros((B, self.nv), tio)
        gc64 = int(Gc is not None and Gc.dtype == np.float64 and pk is not None)
        Gc = pad(_as(Gc, np.float64 if gc64 else np.float32)); hc = pad(_as(hc, np.float64 if gc64 else np.float32))
        pk64 = int(pk is not None and pk.dtype == np.float64)
        if pk is not None:
            pk = np.ascontiguousarray(pk)
            Jd = ed = epd = None
        else:
            Jd, ed = _as(J, np.float32), pad(_as(e, np.float32))
            epd = None if (ep is None or ptgt is not None) else pad(_as(ep, np.float32))
        ptgt = _as(ptgt, tio)
        batched = int(ptgt is not None and ptgt.size == B * s.nposture * self.nq and B > 1)
        if warm is not None:
            assert warm.dtype == np.int8 and warm.flags.c_contiguous
        skip = _as(skip, np.int32)
        self.last_rc = lib().emu_solve(self.h, B, path, int(io64), _vp(q), _vp(pk), pk64, _p(Jd), _p(ed), _p(epd), _vp(ptgt), batched,
                                       _vp(Gc), _vp(hc), gc64, C.c_double(dt), C.c_double(damping), _vp(dq), int(integrate),
                                       _p(st, C.c_int32), _p(it, C.c_int32), _p(H, C.c_double), _p(c, C.c_double), _vp(lo), _vp(hi),
                                       None if warm is None else warm.ctypes.data_as(C.POINTER(C.c_byte)), _p(skip, C.c_int32))
        assert self.last_rc == 0, lib().emu_last_error()
        out = (dq, st, it, H, c, lo, hi)
        return out + (q,) if integrate else out

    def solve_warm(self, q, J, e, ep, dt, damping, dq_prev, warm, use_double=None):
        """One step of a rollout: `warm` ([B, nu] int8, zeros before the first step) and `dq_prev` (the previous step's dq)
        are updated in place, as bik_step does between its steps."""
        if use_double is None:
            use_double = 8 if self.header()["nu"] > 32 else 3
        dq, st, it, *_ = self.solve(q, J, e, ep, None, None, dt, damping, use_double=use_double, warm=warm, dq_inout=dq_prev)
        return dq, st, it

    def _loop_inputs(self, q, ftgt, ptgt, ctgt):
        """q and the targets in q's dtype: float64 runs the ...64 loops, anything else the fp32 ones (as engine.py picks)."""
        t = np.float64 if np.asarray(q).dtype == np.float64 else np.float32
        q = _as(q, t).copy(); B = q.shape[0]
        ftgt, ptgt, ctgt = _as(ftgt, t), _as(ptgt, t), _as(ctgt, t)
        batched = int(ptgt is not None and ptgt.size == B * self.spec.nposture * self.nq and B > 1)
        return int(t == np.float64), q, ftgt, ptgt, ctgt, batched

    def converge(self, q, ftgt, ptgt, ctgt, dt, damping, max_iters, pos_threshold, ori_threshold):
        """The pass loop of bik_converge, or of bik_converge64 for a float64 q.  Returns (q, iters, status)."""
        f64, q, ftgt, ptgt, ctgt, batched = self._loop_inputs(q, ftgt, ptgt, ctgt)
        B = q.shape[0]
        it = np.zeros(B, np.int32); st = np.zeros(B, np.int32)
        rc = lib().emu_converge(self.h, f64, B, _vp(q), _vp(ftgt), _vp(ptgt), batched, _vp(ctgt), C.c_double(dt), C.c_double(damping),
                                int(max_iters), C.c_double(pos_threshold), C.c_double(ori_threshold), _p(it, C.c_int32), _p(st, C.c_int32))
        assert rc == 0, lib().emu_last_error()
        return q, it, st

    def track(self, q, ftgt, ptgt, ctgt, dt, damping, max_iters, pos_threshold, ori_threshold, lengths=None):
        """The pass loop of bik_track, or of bik_track64 for a float64 q: ftgt [B,T,F,7], ctgt [B,T,C,3].  Returns
        (q, q_traj, iters, status, passes); rows past an instance's length hold NaN / -1 / -1."""
        f64, q, ftgt, ptgt, ctgt, batched = self._loop_inputs(q, ftgt, ptgt, ctgt)
        B, T = q.shape[0], (ftgt if ftgt is not None else ctgt).shape[1]
        q_traj = np.full((B, T, self.nq), np.nan, q.dtype)
        it = np.full((B, T), -1, np.int32); st = np.full((B, T), -1, np.int32); passes = np.zeros(1, np.int32)
        ln = _as(lengths, np.int32)
        rc = lib().emu_track(self.h, f64, B, T, _vp(q), _vp(ftgt), _vp(ptgt), batched, _vp(ctgt), _p(ln, C.c_int32), C.c_double(dt),
                             C.c_double(damping), int(max_iters), C.c_double(pos_threshold), C.c_double(ori_threshold), _vp(q_traj),
                             _p(it, C.c_int32), _p(st, C.c_int32), _p(passes, C.c_int32))
        assert rc == 0, lib().emu_last_error()
        return q, q_traj, it, st, int(passes[0])

    def fk(self, q, frames, want_J=False, f64=False):
        t = np.float64 if f64 else np.float32
        q = _as(q, t); B = q.shape[0]
        poses = np.zeros((B, len(frames), 7), t); com = np.zeros((B, 3), t)
        J = np.zeros((B, len(frames), 6, self.nv), t) if want_J else None
        assert lib().emu_fk(self.h, B, int(f64), _vp(q), c_frames(frames), len(frames), _vp(poses), _vp(com), _vp(J)) == 0
        return poses, com, J

    def integrate(self, q, dq, f64=False):
        """integrate_instance<float>, or integrate_instance<double> when f64 (q and dq in that precision)."""
        t = np.float64 if f64 else np.float32
        q, dq = _as(q, t).copy(), _as(dq, t)
        lib().emu_integrate(self.h, int(f64), q.shape[0], _vp(q), _vp(dq))
        return q

    def check_limits(self, q, tol=1e-6):
        q = _as(q, np.float32); st = np.zeros(q.shape[0], np.int32)
        lib().emu_check_limits(self.h, q.shape[0], _p(q), C.c_float(tol), _p(st, C.c_int32))
        return st


# ---- bik_math.h's Lie layer, one function at a time ---------------------------------------------------------------------
# Each takes fp64 arrays with leading batch dimensions, rounds them to the instantiation's type (f64=False: float) and returns
# the results widened to fp64.
def _lie(fn, f64, a, b, out_shape, out2=False):
    a = np.ascontiguousarray(a, np.float64)
    lead = a.shape[:-1]
    n = int(np.prod(lead, dtype=np.int64))
    b = None if b is None else np.ascontiguousarray(np.broadcast_to(b, lead + np.shape(b)[-1:]), np.float64)
    out = np.zeros(lead + out_shape)
    o2 = np.zeros(lead + out_shape) if out2 else None
    assert lib().emu_lie(fn, int(f64), n, _vp(a), _vp(b), _vp(out), _vp(o2)) == 0
    return (out, o2) if out2 else out


def lie_coefs(t2, f64):
    """coef_A and coef_BCD at theta^2 = t2: [..., 4] = (A, B, C, D)."""
    return _lie(0, f64, np.asarray(t2, np.float64)[..., None], None, (4,))


def lie_so3_log(q, f64):
    return _lie(1, f64, q, None, (3,))


def lie_se3_log(q, t, f64):
    """[..., 6] = (v, w)."""
    return _lie(2, f64, q, t, (6,))


def lie_ljacinv_blocks(xi, f64):
    """se3_ljacinv_blocks at xi = (v, w): (Ji, Mi), each [..., 3, 3]."""
    return _lie(3, f64, xi, None, (3, 3), out2=True)


def lie_quat_sub(qa, qb, f64):
    return _lie(4, f64, qa, qb, (3,))


def lie_quat_integrate(q, w, f64):
    return _lie(5, f64, q, w, (4,))
