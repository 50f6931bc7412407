"""Low-level batched engine: thin, typed wrapper over the C ABI using torch CUDA tensors for memory.

`DeviceModel` owns a bik_model, `Problem` a bik_problem.  All methods enqueue kernels on torch's
current stream and return torch tensors on the model's device; nothing here computes -- torch is used
for allocation, streams and host<->device copies only.

Precision follows the dtype of `q`: float32 tensors take the fp32 entry points (the batched fast path),
float64 tensors the ...64 entry points (fp64 kernels end to end, the reference's precision).  numpy inputs
other than q are converted to q's dtype.
"""

from __future__ import annotations

import ctypes as C
from typing import Optional, Sequence

import numpy as np
import torch

from . import _lib
from ._abi import POSTURE_SEQ_BATCHED, POSTURE_SEQ_SHARED, BikBounds, BikCollision, BikDims, BikInputs, ProblemSpec, c_frames
from .flatten import FlatModel, Frame


def _stream() -> int:
    return torch.cuda.current_stream().cuda_stream


def _ptr(t: Optional[torch.Tensor]):
    return None if t is None else t.data_ptr()


def _is64(t: torch.Tensor) -> bool:
    return t.dtype == torch.float64


class DeviceModel:
    def __init__(self, flat: FlatModel, device: Optional[int] = None):
        if not torch.cuda.is_available():
            raise RuntimeError("mink_b200 needs a CUDA device: the IK hot path has no CPU implementation")
        self.flat = flat
        self.device = torch.cuda.current_device() if device is None else int(device)
        self.lib = _lib.load()
        blob = flat.to_blob()
        h = C.c_void_p()
        _lib.check(self.lib.bik_model_create(blob, len(blob), self.device, C.byref(h)))
        self.handle = h
        self.nq, self.nv = flat.nq, flat.nv

    def __del__(self):
        # problems created through tasks.problem_for() reference this model: release them first
        for prob in list(self.__dict__.get("_problems", {}).values()):
            prob.close()
        h, self.handle = getattr(self, "handle", None), None
        if h:
            self.lib.bik_model_destroy(h)

    def _dev(self, a, dtype=None) -> torch.Tensor:
        """Contiguous CUDA tensor of `dtype` (default: float64 tensors stay float64, everything else becomes float32)."""
        if isinstance(a, np.ndarray) and not a.flags.writeable:
            a = a.copy()
        t = torch.as_tensor(a)
        if dtype is None:
            dtype = torch.float64 if (isinstance(a, torch.Tensor) and a.dtype == torch.float64) else torch.float32
        return t.to(device=f"cuda:{self.device}", dtype=dtype).contiguous()

    def _rows(self, a, *tail, dtype=None) -> torch.Tensor:
        """CUDA tensor viewed as [-1, *tail] (well defined for empty batches too)."""
        t = self._dev(a, dtype)
        n = 1
        for d in tail:
            n *= d
        return t.reshape((t.numel() // n,) + tuple(tail))

    def fk(self, q, frames: Sequence[Frame], want_com: bool = False):
        q = self._rows(q, self.nq)
        B, F = q.shape[0], len(frames)
        poses = torch.empty((B, F, 7), device=q.device, dtype=q.dtype)
        com = torch.empty((B, 3), device=q.device, dtype=q.dtype) if want_com else None
        fn = self.lib.bik_fk64 if _is64(q) else self.lib.bik_fk
        _lib.check(fn(self.handle, B, q.data_ptr(), c_frames(frames), F, poses.data_ptr(), _ptr(com), _stream()))
        return poses, com

    def frame_jacobian(self, q, frames: Sequence[Frame]):
        q = self._rows(q, self.nq)
        B, F = q.shape[0], len(frames)
        J = torch.empty((B, F, 6, self.nv), device=q.device, dtype=q.dtype)
        fn = self.lib.bik_frame_jacobian64 if _is64(q) else self.lib.bik_frame_jacobian
        _lib.check(fn(self.handle, B, q.data_ptr(), c_frames(frames), F, J.data_ptr(), _stream()))
        return J

    def integrate(self, q: torch.Tensor, dq: torch.Tensor) -> torch.Tensor:
        """In place on q ([B,nq] CUDA, fp32 or fp64; dq is converted to q's dtype)."""
        dq = dq.to(q.dtype).reshape(-1, self.nv)
        if dq.shape[0] != q.shape[0]:
            if dq.shape[0] != 1:
                raise ValueError(f"velocity batch {dq.shape[0]} does not match the configuration batch {q.shape[0]}")
            dq = dq.expand(q.shape[0], -1)
        dq = dq.contiguous()
        fn = self.lib.bik_integrate64 if _is64(q) else self.lib.bik_integrate
        _lib.check(fn(self.handle, q.shape[0], q.data_ptr(), dq.data_ptr(), _stream()))
        return q

    def check_limits(self, q: torch.Tensor, tol: float = 1e-6) -> torch.Tensor:
        st = torch.empty(q.shape[0], device=q.device, dtype=torch.int32)
        fn = self.lib.bik_check_limits64 if _is64(q) else self.lib.bik_check_limits
        _lib.check(fn(self.handle, q.shape[0], q.data_ptr(), float(tol), st.data_ptr(), _stream()))
        return st


class Problem:
    def __init__(self, model: DeviceModel, spec: ProblemSpec):
        self.model, self.spec, self.lib = model, spec, model.lib
        t, nt, l, nl, self._keep = spec.to_c()
        h = C.c_void_p()
        _lib.check(self.lib.bik_problem_create(model.handle, t, nt, l, nl, C.byref(h)))
        self.handle = h
        d = BikDims()
        _lib.check(self.lib.bik_problem_dims(h, C.byref(d)))
        self.nq, self.nv, self.F, self.P, self.Cn, self.K, self.npairs = d.nq, d.nv, d.nframe, d.nposture, d.ncom, d.nrows, d.npairs

    def describe(self, damping: float = 1e-12) -> str:
        """How the problem is mapped onto the device (K1 lanes and precision, coupled block, K2 path); bik_problem_describe."""
        buf = C.create_string_buffer(768)
        self.lib.bik_problem_describe(self.handle, float(damping), buf, 768)
        return buf.value.decode()

    def close(self):
        h, self.handle = getattr(self, "handle", None), None
        if h:
            self.lib.bik_problem_destroy(h)

    def __del__(self):
        self.close()

    # -- inputs --------------------------------------------------------------------------------
    def _inputs(self, q, frame_targets, posture_targets, com_targets, dtype=None):
        """bik_inputs for one call.  The element type is q's (or `dtype` when q is passed separately)."""
        m = self.model
        keep = []
        inp = BikInputs()
        B = None
        if q is not None:
            q = m._rows(q, self.nq)
            dtype = q.dtype
            B = q.shape[0]
            inp.q = q.data_ptr()
            keep.append(q)
        dtype = dtype or torch.float32
        inp.f64 = int(dtype == torch.float64)
        if self.F:
            if frame_targets is None:
                raise ValueError("No target set for FrameTask")
            ft = m._rows(frame_targets, self.F, 7, dtype=dtype)
            inp.frame_targets = ft.data_ptr()
            keep.append(ft)
            B = ft.shape[0] if B is None else B
        if self.P:
            if posture_targets is None:
                raise ValueError("No target set for PostureTask")
            pt = m._rows(posture_targets, self.P, self.nq, dtype=dtype)
            inp.posture_targets = pt.data_ptr()
            inp.posture_batched = int(pt.shape[0] > 1)
            keep.append(pt)
        if self.Cn:
            if com_targets is None:
                raise ValueError("No target set for ComTask")
            ct = m._rows(com_targets, self.Cn, 3, dtype=dtype)
            inp.com_targets = ct.data_ptr()
            keep.append(ct)
        return inp, keep, B, q

    def _weights(self, weights, q: torch.Tensor, *lead):
        """Per-instance task weights as a contiguous [*lead, K] CUDA tensor of q's dtype (None stays None)."""
        if weights is None:
            return None
        w = self.model._dev(weights, dtype=q.dtype)
        if tuple(w.shape) != tuple(lead) + (self.K,):
            raise ValueError(f"weights must have shape {tuple(lead) + (self.K,)} (rows of the stacked task Jacobian), got {tuple(w.shape)}")
        return w

    def _posture_weights(self, posture_weights, q: torch.Tensor, *lead):
        """Per-instance posture weights as a contiguous [*lead, P, nv] CUDA tensor of q's dtype (None stays None)."""
        if posture_weights is None:
            return None
        if not self.P:
            raise ValueError("posture_weights given for a problem without a PostureTask or DampingTask")
        w = self.model._dev(posture_weights, dtype=q.dtype)
        if tuple(w.shape) != tuple(lead) + (self.P, self.nv):
            raise ValueError(f"posture_weights must have shape {tuple(lead) + (self.P, self.nv)} (posture-type tasks x dofs), got {tuple(w.shape)}")
        return w

    def _bounds(self, bounds, q: torch.Tensor, B: int):
        """Per-instance bounds (lower, upper, vmax) as a BikBounds of contiguous [B, nv] CUDA tensors of q's dtype, and the
        tensors it points to; None for no bounds or three Nones (the call then runs the ..._weighted_ex entry point)."""
        if bounds is None or all(x is None for x in bounds):
            return None, []
        if len(bounds) != 3:
            raise ValueError("bounds must be a (lower, upper, vmax) tuple, each [B, nv] or None")
        keep, out = [], BikBounds()
        for name, x in zip(("lower", "upper", "vmax"), bounds):
            if x is None:
                continue
            t = self.model._dev(x, dtype=q.dtype)
            if tuple(t.shape) != (B, self.nv):
                raise ValueError(f"bounds {name} must have shape {(B, self.nv)} (instances x dofs), got {tuple(t.shape)}")
            keep.append(t)
            setattr(out, name, t.data_ptr())
        return out, keep

    def _collision(self, collision, q: torch.Tensor, B: int, T: Optional[int] = None):
        """Per-instance collision arguments (enabled, minimum_distance, detection_distance) as a BikCollision of contiguous CUDA
        tensors, and the tensors it points to: enabled [B, npairs] (track: [B, T, npairs]) as uint8, the distances [B] (track:
        [B, T]) in q's dtype.  None for None or three Nones (the call then runs the ..._bounded entry point)."""
        if collision is None or all(x is None for x in collision):
            return None, []
        if len(collision) != 3:
            raise ValueError("collision must be an (enabled, minimum_distance, detection_distance) tuple, each a tensor or None")
        lead = (B,) if T is None else (B, T)
        keep, out = [], BikCollision()
        for name, x in zip(("enabled", "minimum_distance", "detection_distance"), collision):
            if x is None:
                continue
            shape = lead + (self.npairs,) if name == "enabled" else lead
            t = self.model._dev(x, dtype=torch.uint8 if name == "enabled" else q.dtype)
            if tuple(t.shape) != shape:
                raise ValueError(f"collision {name} must have shape {shape}, got {tuple(t.shape)}")
            keep.append(t)
            setattr(out, name, t.data_ptr())
        return out, keep

    def _placement(self, placement, q: torch.Tensor, B: int):
        """Per-instance frame placements as a contiguous [B, F, 7] CUDA tensor of q's dtype (None stays None)."""
        if placement is None:
            return None
        if not self.F:
            raise ValueError("placement given for a problem without a FrameTask or RelativeFrameTask")
        t = self.model._dev(placement, dtype=q.dtype)
        if tuple(t.shape) != (B, self.F, 7):
            raise ValueError(f"placement must have shape {(B, self.F, 7)} (instances x frame tasks x wxyz_xyz), got {tuple(t.shape)}")
        return t

    def fk_jac(self, q, frame_targets=None, posture_targets=None, com_targets=None, dt: float = 1e-2):
        inp, keep, B, q = self._inputs(q, frame_targets, posture_targets, com_targets)
        dev, dt_ = q.device, q.dtype
        J = torch.empty((B, self.K, self.nv), device=dev, dtype=dt_)
        e = torch.empty((B, self.K), device=dev, dtype=dt_)
        ep = torch.empty((B, self.P, self.nv), device=dev, dtype=dt_)
        Gc = torch.empty((B, self.npairs, self.nv), device=dev, dtype=dt_)
        hc = torch.empty((B, self.npairs), device=dev, dtype=dt_)
        fn = self.lib.bik_fk_jac64 if _is64(q) else self.lib.bik_fk_jac
        _lib.check(fn(self.handle, B, C.byref(inp), float(dt), _ptr(J) if self.K else None,
                      _ptr(e) if self.K else None, _ptr(ep) if self.P else None,
                      _ptr(Gc) if self.npairs else None, _ptr(hc) if self.npairs else None, _stream()))
        return J, e, ep, Gc, hc

    def objective(self, J, e, ep, damping: float):
        ref = J if self.K else ep
        B, dev = ref.shape[0], ref.device
        H = torch.empty((B, self.nv, self.nv), device=dev, dtype=torch.float64)
        c = torch.empty((B, self.nv), device=dev, dtype=torch.float64)
        fn = self.lib.bik_qp_objective64 if _is64(ref) else self.lib.bik_qp_objective
        _lib.check(fn(self.handle, B, _ptr(J) if self.K else None, _ptr(e) if self.K else None,
                      _ptr(ep) if self.P else None, float(damping), H.data_ptr(), c.data_ptr(), _stream()))
        return H, c

    def box(self, q, dt: float):
        q = self.model._rows(q, self.nq)
        lo = torch.empty((q.shape[0], self.nv), device=q.device, dtype=q.dtype)
        hi = torch.empty_like(lo)
        fn = self.lib.bik_limits_box64 if _is64(q) else self.lib.bik_limits_box
        _lib.check(fn(self.handle, q.shape[0], q.data_ptr(), float(dt), lo.data_ptr(), hi.data_ptr(), _stream()))
        return lo, hi

    def solve(self, q, J, e, ep, Gc, hc, dt: float, damping: float, return_iters: bool = False):
        """K2 alone on dense task rows (J, e, e_posture, collision rows must have q's dtype)."""
        q = self.model._rows(q, self.nq)
        B = q.shape[0]
        for t in (J, e, ep, Gc, hc):
            assert t is None or t.numel() == 0 or t.dtype == q.dtype, "task rows and q must share their dtype"
        dq = torch.empty((B, self.nv), device=q.device, dtype=q.dtype)
        st = torch.empty(B, device=q.device, dtype=torch.int32)
        it = torch.zeros(B, device=q.device, dtype=torch.int32) if return_iters else None
        args = (self.handle, B, q.data_ptr(), _ptr(J) if self.K else None, _ptr(e) if self.K else None,
                _ptr(ep) if self.P else None, _ptr(Gc) if self.npairs else None,
                _ptr(hc) if self.npairs else None, float(dt), float(damping), dq.data_ptr(), st.data_ptr(), _ptr(it), _stream())
        _lib.check(self.lib.bik_solve64(*args) if _is64(q) else self.lib.bik_solve_ex(*args))
        return (dq, st, it) if return_iters else (dq, st)

    def step(self, q: torch.Tensor, frame_targets=None, posture_targets=None, com_targets=None, dt: float = 1e-2,
             damping: float = 1e-12, nsteps: int = 1, integrate: bool = False, dq: Optional[torch.Tensor] = None,
             status: Optional[torch.Tensor] = None, weights=None, posture_weights=None, bounds=None, collision=None, placement=None):
        """solve_ik (x nsteps, optionally integrating q in place).  q: [B,nq] fp32 or fp64 CUDA tensor.
        weights: [B, K] per-instance multipliers in [0, 1] of the frame / CoM task costs, rows in the stacked order of J
        (bik_step_weighted); None: the problem's costs.
        posture_weights: [B, P, nv] per-instance multipliers in [0, 1] of the PostureTask / DampingTask dof costs, tasks in the
        order of the posture targets (bik_step_weighted_ex); None: the problem's costs.
        bounds: (lower, upper, vmax), each [B, nv] (tangent dofs) or None, that narrow the problem's ConfigurationLimit bounds
        and VelocityLimit caps per instance on the dofs those limits list (bik_step_bounded; bik.h); None: the problem's.
        collision: (enabled, minimum_distance, detection_distance), each None or enabled [B, npairs] (pair k of instance b is
        used iff != 0) and the distances [B], that replace the CollisionAvoidanceLimit's pairs and distances per instance
        (bik_step_coll; bik.h); None: the problem's.
        placement: [B, F, 7] per-instance poses (wxyz_xyz) of the frame tasks' frames in their tree nodes, tasks in the order of
        the frame targets, in place of the problem's (bik_step_placed; bik.h); None: the problem's."""
        assert q.is_cuda and q.dtype in (torch.float32, torch.float64) and q.is_contiguous()
        inp, keep, _, _ = self._inputs(None, frame_targets, posture_targets, com_targets, dtype=q.dtype)
        B = q.shape[0]
        w = self._weights(weights, q, B)
        pw = self._posture_weights(posture_weights, q, B)
        bd, keep_bd = self._bounds(bounds, q, B)
        co, keep_co = self._collision(collision, q, B)
        pl = self._placement(placement, q, B)
        if dq is None:
            dq = torch.empty((B, self.nv), device=q.device, dtype=q.dtype)
        if status is None:
            status = torch.empty(B, device=q.device, dtype=torch.int32)
        assert dq.dtype == q.dtype
        args = (float(dt), float(damping), int(nsteps), int(bool(integrate)), dq.data_ptr(), status.data_ptr(), _stream())
        if pl is not None:
            fn = self.lib.bik_step_placed64 if _is64(q) else self.lib.bik_step_placed
            _lib.check(fn(self.handle, B, q.data_ptr(), C.byref(inp), _ptr(w), _ptr(pw), None if bd is None else C.byref(bd),
                          None if co is None else C.byref(co), pl.data_ptr(), *args))
        elif co is not None:
            fn = self.lib.bik_step_coll64 if _is64(q) else self.lib.bik_step_coll
            _lib.check(fn(self.handle, B, q.data_ptr(), C.byref(inp), _ptr(w), _ptr(pw), None if bd is None else C.byref(bd), C.byref(co), *args))
        elif bd is not None:
            fn = self.lib.bik_step_bounded64 if _is64(q) else self.lib.bik_step_bounded
            _lib.check(fn(self.handle, B, q.data_ptr(), C.byref(inp), _ptr(w), _ptr(pw), C.byref(bd), *args))
        elif pw is not None:
            fn = self.lib.bik_step_weighted_ex64 if _is64(q) else self.lib.bik_step_weighted_ex
            _lib.check(fn(self.handle, B, q.data_ptr(), C.byref(inp), _ptr(w), pw.data_ptr(), *args))
        elif w is None:
            fn = self.lib.bik_step64 if _is64(q) else self.lib.bik_step
            _lib.check(fn(self.handle, B, q.data_ptr(), C.byref(inp), *args))
        else:
            fn = self.lib.bik_step_weighted64 if _is64(q) else self.lib.bik_step_weighted
            _lib.check(fn(self.handle, B, q.data_ptr(), C.byref(inp), w.data_ptr(), *args))
        return dq, status

    def converge(self, q: torch.Tensor, frame_targets=None, posture_targets=None, com_targets=None, dt: float = 1e-2,
                 damping: float = 1e-12, max_iters: int = 20, pos_threshold: float = 1e-4, ori_threshold: float = 1e-4,
                 check_every: int = 1, weights=None, posture_weights=None, bounds=None, collision=None, placement=None):
        """solve_ik + integrate until every frame task is within the thresholds or max_iters steps were taken, per instance
        (the inner loop of the reference's examples; bik_converge for a float32 q, bik_converge64 for a float64 q, the
        targets in q's dtype).  q is updated in place.  weights: [B, K] as in `step` (bik_converge_weighted); a frame task
        whose three position (orientation) weights are 0 is left out of the position (orientation) test.
        posture_weights: [B, P, nv] as in `step` (bik_converge_weighted_ex).  bounds: as in `step` (bik_converge_bounded).
        collision: as in `step` (bik_converge_coll).  placement: [B, F, 7] as in `step` (bik_converge_placed).
        Returns (iters [B], status [B])."""
        assert q.is_cuda and q.dtype in (torch.float32, torch.float64) and q.is_contiguous()
        inp, keep, _, _ = self._inputs(None, frame_targets, posture_targets, com_targets, dtype=q.dtype)
        B = q.shape[0]
        w = self._weights(weights, q, B)
        pw = self._posture_weights(posture_weights, q, B)
        bd, keep_bd = self._bounds(bounds, q, B)
        co, keep_co = self._collision(collision, q, B)
        pl = self._placement(placement, q, B)
        iters = torch.zeros(B, device=q.device, dtype=torch.int32)
        status = torch.zeros(B, device=q.device, dtype=torch.int32)
        args = (float(dt), float(damping), int(max_iters), float(pos_threshold), float(ori_threshold), int(check_every), iters.data_ptr(),
                status.data_ptr(), _stream())
        if pl is not None:
            fn = self.lib.bik_converge_placed64 if _is64(q) else self.lib.bik_converge_placed
            _lib.check(fn(self.handle, B, q.data_ptr(), C.byref(inp), _ptr(w), _ptr(pw), None if bd is None else C.byref(bd),
                          None if co is None else C.byref(co), pl.data_ptr(), *args))
        elif co is not None:
            fn = self.lib.bik_converge_coll64 if _is64(q) else self.lib.bik_converge_coll
            _lib.check(fn(self.handle, B, q.data_ptr(), C.byref(inp), _ptr(w), _ptr(pw), None if bd is None else C.byref(bd), C.byref(co), *args))
        elif bd is not None:
            fn = self.lib.bik_converge_bounded64 if _is64(q) else self.lib.bik_converge_bounded
            _lib.check(fn(self.handle, B, q.data_ptr(), C.byref(inp), _ptr(w), _ptr(pw), C.byref(bd), *args))
        elif pw is not None:
            fn = self.lib.bik_converge_weighted_ex64 if _is64(q) else self.lib.bik_converge_weighted_ex
            _lib.check(fn(self.handle, B, q.data_ptr(), C.byref(inp), _ptr(w), pw.data_ptr(), *args))
        elif w is None:
            fn = self.lib.bik_converge64 if _is64(q) else self.lib.bik_converge
            _lib.check(fn(self.handle, B, q.data_ptr(), C.byref(inp), *args))
        else:
            fn = self.lib.bik_converge_weighted64 if _is64(q) else self.lib.bik_converge_weighted
            _lib.check(fn(self.handle, B, q.data_ptr(), C.byref(inp), w.data_ptr(), *args))
        return iters, status

    def track(self, q: torch.Tensor, frame_targets=None, posture_targets=None, com_targets=None, lengths=None, dt: float = 1e-2,
              damping: float = 1e-12, max_iters: int = 20, pos_threshold: float = 1e-4, ori_threshold: float = 1e-4,
              check_every: int = 1, weights=None, posture_seq: bool = False, posture_weights=None, bounds=None, collision=None,
              hold=None, placement=None):
        """The converge loop over a sequence of targets, each instance on its own frame cursor (bik_track for a float32 q,
        bik_track64 for a float64 q; the targets and q_traj in q's dtype):
        for every instance b and frame t < lengths[b] (default: all T), what `converge` on frame t's targets gives.
        frame_targets [B,T,F,7], com_targets [B,T,C,3]; posture targets as in `converge` (the same for every frame), or with
        posture_seq=True a sequence: [T,P,nq] shared by the batch or [B,T,P,nq] per instance.
        q [B,nq] is updated in place to the end of each instance's last frame.
        Returns (q_traj [B,T,nq], iters [B,T], status [B,T], passes): rows past an instance's length hold NaN / -1 / -1;
        passes is a 0-d tensor, the number of passes the device loop ran.
        weights: [B, T, K] per-frame task weights as in `converge` (bik_track_weighted), or None.
        posture_weights: [B, T, P, nv] per-frame posture weights as in `converge` (bik_track_weighted_ex), or None.
        bounds: as in `converge`, [B, nv] each, one row per instance for every frame (bik_track_bounded), or None.
        collision: as in `converge` with one row per instance and frame, enabled [B, T, npairs] and the distances [B, T]
        (bik_track_coll), or None.
        hold: [B, T, H] bools, H = F + C + P: the frame-like tasks, then the CoM tasks, then the posture-type tasks, each in
        the order of its targets (bik_track_hold), or None.  Over a run of frames where hold[b, :, k] is set, task k's target
        is its value at the configuration instance b had when the run began (set_target_from_configuration), captured on the
        device; its target rows on those frames are ignored.
        placement: [B, F, 7] as in `converge`, one row per instance for every frame (bik_track_placed), or None."""
        assert q.is_cuda and q.dtype in (torch.float32, torch.float64) and q.is_contiguous()
        m = self.model
        B = q.shape[0]
        seqs = [m._rows(t, n, k, dtype=q.dtype) for t, n, k in ((frame_targets, self.F, 7), (com_targets, self.Cn, 3))
                if n and t is not None]
        if not seqs:
            raise ValueError("bik_track needs frame or CoM target sequences to take the number of frames from")
        T = seqs[0].shape[0] // max(B, 1)
        for s in seqs:
            if B == 0 or s.shape[0] != B * T or T < 1:
                raise ValueError(f"target sequences must be [B={B}, T, ...] with the same T >= 1")
        inp, keep, _, _ = self._inputs(None, frame_targets, posture_targets, com_targets, dtype=q.dtype)
        if posture_seq and self.P:
            n = keep[1 if self.F else 0].numel()   # (_inputs keeps the frame, posture, CoM targets in that order)
            if n not in (T * self.P * self.nq, B * T * self.P * self.nq):
                raise ValueError(f"a posture target sequence must be [T={T}, P={self.P}, nq={self.nq}] or [B={B}, T, P, nq]")
            inp.posture_batched = POSTURE_SEQ_SHARED if n == T * self.P * self.nq else POSTURE_SEQ_BATCHED
        w = self._weights(weights, q, B, T)
        pw = self._posture_weights(posture_weights, q, B, T)
        bd, keep_bd = self._bounds(bounds, q, B)
        co, keep_co = self._collision(collision, q, B, T)
        hd = None
        if hold is not None:
            H = self.F + self.Cn + self.P
            hd = m._dev(hold, torch.uint8)
            if hd.shape != (B, T, H):
                raise ValueError(f"hold must be [B={B}, T={T}, H={H}] (frame, CoM and posture-type tasks), not {list(hd.shape)}")
        pl = self._placement(placement, q, B)
        ln = None
        if lengths is not None:
            ln = m._dev(lengths, torch.int32).reshape(-1)
            if ln.shape[0] != B:
                raise ValueError(f"lengths has {ln.shape[0]} entries for a batch of {B}")
        q_traj = torch.full((B, T, self.nq), float("nan"), device=q.device, dtype=q.dtype)
        iters = torch.full((B, T), -1, device=q.device, dtype=torch.int32)
        status = torch.full((B, T), -1, device=q.device, dtype=torch.int32)
        passes = torch.zeros(1, device=q.device, dtype=torch.int32)
        args = (_ptr(ln), float(dt), float(damping), int(max_iters), float(pos_threshold), float(ori_threshold), int(check_every),
                q_traj.data_ptr(), iters.data_ptr(), status.data_ptr(), passes.data_ptr(), _stream())
        if pl is not None:
            fn = self.lib.bik_track_placed64 if _is64(q) else self.lib.bik_track_placed
            _lib.check(fn(self.handle, B, T, q.data_ptr(), C.byref(inp), _ptr(w), _ptr(pw), None if bd is None else C.byref(bd),
                          None if co is None else C.byref(co), _ptr(hd), pl.data_ptr(), *args))
        elif hd is not None:
            fn = self.lib.bik_track_hold64 if _is64(q) else self.lib.bik_track_hold
            _lib.check(fn(self.handle, B, T, q.data_ptr(), C.byref(inp), _ptr(w), _ptr(pw), None if bd is None else C.byref(bd),
                          None if co is None else C.byref(co), hd.data_ptr(), *args))
        elif co is not None:
            fn = self.lib.bik_track_coll64 if _is64(q) else self.lib.bik_track_coll
            _lib.check(fn(self.handle, B, T, q.data_ptr(), C.byref(inp), _ptr(w), _ptr(pw), None if bd is None else C.byref(bd), C.byref(co), *args))
        elif bd is not None:
            fn = self.lib.bik_track_bounded64 if _is64(q) else self.lib.bik_track_bounded
            _lib.check(fn(self.handle, B, T, q.data_ptr(), C.byref(inp), _ptr(w), _ptr(pw), C.byref(bd), *args))
        elif pw is not None:
            fn = self.lib.bik_track_weighted_ex64 if _is64(q) else self.lib.bik_track_weighted_ex
            _lib.check(fn(self.handle, B, T, q.data_ptr(), C.byref(inp), _ptr(w), pw.data_ptr(), *args))
        elif w is None:
            fn = self.lib.bik_track64 if _is64(q) else self.lib.bik_track
            _lib.check(fn(self.handle, B, T, q.data_ptr(), C.byref(inp), *args))
        else:
            fn = self.lib.bik_track_weighted64 if _is64(q) else self.lib.bik_track_weighted
            _lib.check(fn(self.handle, B, T, q.data_ptr(), C.byref(inp), w.data_ptr(), *args))
        return q_traj, iters, status, passes[0]

    def step_host(self, q: np.ndarray, frame_targets=None, posture_targets=None, com_targets=None, dt: float = 1e-2,
                  damping: float = 1e-12, nsteps: int = 1, integrate: bool = False, out_dq: np.ndarray = None,
                  out_status: np.ndarray = None):
        """Host-buffer entry (numpy fp32 in, numpy fp32 out; copies inside).  `q` is updated in place when
        integrating.  Pass page-locked arrays (e.g. torch pinned tensors' .numpy()) for full copy bandwidth.
        Returns (dq, status, q, h2d_bytes, d2h_bytes)."""
        f32 = lambda a: None if a is None else np.ascontiguousarray(a, dtype=np.float32)
        q = f32(q).reshape(-1, self.nq)
        B = q.shape[0]
        ft, pt, ct = f32(frame_targets), f32(posture_targets), f32(com_targets)
        inp = BikInputs()
        if self.F:
            inp.frame_targets = ft.ctypes.data
        if self.P:
            inp.posture_targets = pt.ctypes.data
            inp.posture_batched = int(pt.size == B * self.P * self.nq and B > 1)
        if self.Cn:
            inp.com_targets = ct.ctypes.data
        dq = out_dq if out_dq is not None else np.empty((B, self.nv), np.float32)
        st = out_status if out_status is not None else np.empty(B, np.int32)
        assert dq.dtype == np.float32 and dq.flags.c_contiguous and st.dtype == np.int32
        up, down = C.c_size_t(0), C.c_size_t(0)
        _lib.check(self.lib.bik_step_host(self.handle, B, q.ctypes.data, C.byref(inp), float(dt), float(damping), int(nsteps),
                                          int(bool(integrate)), dq.ctypes.data, st.ctypes.data, C.byref(up), C.byref(down)))
        return dq, st, q, int(up.value), int(down.value)
