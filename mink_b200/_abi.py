"""ctypes mirror of include/bik.h (struct layouts + descriptor builders).

Pure interface definitions: no compute.  `ProblemSpec` is the host-side, library-independent
description of a task/limit layout; `.to_c()` lowers it to the bik_task_desc / bik_limit_desc
arrays of the C ABI (keeping the backing numpy buffers alive).
"""

from __future__ import annotations

import ctypes as C
from dataclasses import dataclass, field
from typing import List, Optional, Sequence

import numpy as np

from .flatten import FlatModel, Frame

TASK_FRAME, TASK_POSTURE, TASK_COM, TASK_RELATIVE_FRAME = 0, 1, 2, 3
LIMIT_CONFIGURATION, LIMIT_VELOCITY, LIMIT_COLLISION = 0, 1, 2
GEOM_PLANE, GEOM_SPHERE, GEOM_CAPSULE, GEOM_BOX = 0, 2, 3, 6

STATUS_OUT_OF_LIMITS, STATUS_QP_MAXITER, STATUS_NONFINITE, STATUS_QP_INFEASIBLE = 1, 2, 4, 8

# BikInputs.posture_batched: [P][nq], [B][P][nq], and the sequences of the bik_track entry points, [T][P][nq] / [B][T][P][nq]
POSTURE_SHARED, POSTURE_BATCHED, POSTURE_SEQ_SHARED, POSTURE_SEQ_BATCHED = 0, 1, 2, 3

_pd = C.POINTER(C.c_double)
_pi = C.POINTER(C.c_int32)
_pf = C.POINTER(C.c_float)


class BikFrame(C.Structure):
    _fields_ = [("node", C.c_int32), ("reserved", C.c_int32), ("pos", C.c_double * 3), ("quat", C.c_double * 4)]


class BikTaskDesc(C.Structure):
    _fields_ = [("kind", C.c_int32), ("reserved", C.c_int32), ("frame", BikFrame), ("cost", C.c_double * 6),
                ("dof_cost", _pd), ("gain", C.c_double), ("lm_damping", C.c_double), ("root", BikFrame)]


class BikGeom(C.Structure):
    _fields_ = [("type", C.c_int32), ("reserved", C.c_int32), ("frame", BikFrame), ("size", C.c_double * 3)]


class BikLimitDesc(C.Structure):
    _fields_ = [("kind", C.c_int32), ("n", C.c_int32), ("dof", _pi), ("lower", _pd), ("upper", _pd),
                ("vmax", _pd), ("gain", C.c_double), ("geoms", C.POINTER(BikGeom)), ("ngeoms", C.c_int32),
                ("reserved", C.c_int32), ("pairs", _pi), ("minimum_distance", C.c_double),
                ("detection_distance", C.c_double), ("bound_relaxation", C.c_double)]


class BikInputs(C.Structure):
    _fields_ = [("q", C.c_void_p), ("frame_targets", C.c_void_p), ("posture_targets", C.c_void_p),
                ("com_targets", C.c_void_p), ("posture_batched", C.c_int32), ("f64", C.c_int32)]


class BikBounds(C.Structure):   # per-instance bounds of the ..._bounded entry points: [B][nv] device buffers or NULL
    _fields_ = [("lower", C.c_void_p), ("upper", C.c_void_p), ("vmax", C.c_void_p)]


class BikCollision(C.Structure):   # per-instance collision pairs and distances of the ..._coll entry points: device buffers or NULL
    _fields_ = [("enabled", C.c_void_p), ("minimum_distance", C.c_void_p), ("detection_distance", C.c_void_p)]


class BikDims(C.Structure):
    _fields_ = [("nq", C.c_int32), ("nv", C.c_int32), ("nnode", C.c_int32), ("nframe", C.c_int32),
                ("nposture", C.c_int32), ("ncom", C.c_int32), ("nrows", C.c_int32), ("npairs", C.c_int32)]


def c_frame(f: Frame) -> BikFrame:
    out = BikFrame()
    out.node = int(f.node)
    out.pos[:] = [float(x) for x in f.pos]
    out.quat[:] = [float(x) for x in f.quat]
    return out


def c_frames(frames: Sequence[Frame]):
    arr = (BikFrame * max(len(frames), 1))()
    for i, f in enumerate(frames):
        arr[i] = c_frame(f)
    return arr


@dataclass
class TaskSpec:
    kind: int
    frame: Optional[Frame] = None
    cost: np.ndarray = field(default_factory=lambda: np.zeros(6))
    dof_cost: Optional[np.ndarray] = None
    gain: float = 1.0
    lm_damping: float = 0.0
    root: Optional[Frame] = None   # RELATIVE_FRAME


@dataclass
class LimitSpec:
    kind: int
    dof: Optional[np.ndarray] = None
    lower: Optional[np.ndarray] = None
    upper: Optional[np.ndarray] = None
    vmax: Optional[np.ndarray] = None
    gain: float = 0.95
    geoms: Optional[list] = None        # list of (type, Frame, size[3])
    pairs: Optional[np.ndarray] = None  # [n,2] indices into geoms
    minimum_distance: float = 0.005
    detection_distance: float = 0.01
    bound_relaxation: float = 0.0


@dataclass
class ProblemSpec:
    tasks: List[TaskSpec]
    limits: List[LimitSpec]

    @property
    def nframe(self):
        return sum(t.kind in (TASK_FRAME, TASK_RELATIVE_FRAME) for t in self.tasks)

    @property
    def nposture(self):
        return sum(t.kind == TASK_POSTURE for t in self.tasks)

    @property
    def ncom(self):
        return sum(t.kind == TASK_COM for t in self.tasks)

    @property
    def nrows(self):
        return 6 * self.nframe + 3 * self.ncom

    @property
    def npairs(self):
        return sum(len(l.pairs) for l in self.limits if l.kind == LIMIT_COLLISION)

    def key(self) -> bytes:
        """Hashable fingerprint of the static layout (used to cache bik_problem handles)."""
        parts = []
        for t in self.tasks:
            parts.append(np.array([t.kind, t.gain, t.lm_damping], dtype=np.float64).tobytes())
            parts.append(np.asarray(t.cost, dtype=np.float64).tobytes())
            for fr in (t.frame, t.root):
                if fr is not None:
                    parts.append(np.concatenate([[fr.node], fr.pos, fr.quat]).astype(np.float64).tobytes())
            if t.dof_cost is not None:
                parts.append(np.asarray(t.dof_cost, dtype=np.float64).tobytes())
        for l in self.limits:
            parts.append(np.array([l.kind, l.gain, l.minimum_distance, l.detection_distance,
                                   l.bound_relaxation], dtype=np.float64).tobytes())
            for a in (l.dof, l.lower, l.upper, l.vmax, l.pairs):
                if a is not None:
                    parts.append(np.asarray(a, dtype=np.float64).tobytes())
            for g in (l.geoms or []):
                parts.append(np.concatenate([[g[0], g[1].node], g[1].pos, g[1].quat, g[2]]).astype(np.float64).tobytes())
        return b"|".join(parts)

    def to_c(self):
        """-> (tasks array, ntasks, limits array, nlimits, keepalive list)."""
        keep = []
        tarr = (BikTaskDesc * max(len(self.tasks), 1))()
        for i, t in enumerate(self.tasks):
            d = tarr[i]
            d.kind = t.kind
            if t.frame is not None:
                d.frame = c_frame(t.frame)
            if t.root is not None:
                d.root = c_frame(t.root)
            d.cost[:] = [float(x) for x in np.asarray(t.cost, dtype=np.float64)]
            if t.dof_cost is not None:
                buf = np.ascontiguousarray(t.dof_cost, dtype=np.float64)
                keep.append(buf)
                d.dof_cost = buf.ctypes.data_as(_pd)
            d.gain = float(t.gain)
            d.lm_damping = float(t.lm_damping)
        larr = (BikLimitDesc * max(len(self.limits), 1))()
        for i, l in enumerate(self.limits):
            d = larr[i]
            d.kind = l.kind
            d.gain = float(l.gain)
            if l.kind == LIMIT_COLLISION:
                garr = (BikGeom * max(len(l.geoms), 1))()
                for k, (gt, gf, gs) in enumerate(l.geoms):
                    garr[k].type = int(gt)
                    garr[k].frame = c_frame(gf)
                    garr[k].size[:] = [float(x) for x in gs]
                pairs = np.ascontiguousarray(l.pairs, dtype=np.int32).reshape(-1, 2)
                keep += [garr, pairs]
                d.n = pairs.shape[0]
                d.geoms, d.ngeoms = garr, len(l.geoms)
                d.pairs = pairs.ctypes.data_as(_pi)
                d.minimum_distance = float(l.minimum_distance)
                d.detection_distance = float(l.detection_distance)
                d.bound_relaxation = float(l.bound_relaxation)
            else:
                dof = np.ascontiguousarray(l.dof, dtype=np.int32)
                keep.append(dof)
                d.n = dof.shape[0]
                d.dof = dof.ctypes.data_as(_pi)
                for name in ("lower", "upper", "vmax"):
                    a = getattr(l, name)
                    if a is not None:
                        buf = np.ascontiguousarray(a, dtype=np.float64)
                        keep.append(buf)
                        setattr(d, name, buf.ctypes.data_as(_pd))
        return tarr, len(self.tasks), larr, len(self.limits), keep


# --------------------------------------------------------------------------- #
# Workload dictionaries (mink_b200.workloads) -> ProblemSpec.
# --------------------------------------------------------------------------- #
def _collision_pairs(fm: FlatModel, groups, names: List[str]):
    """Geom id pairs after the reference's filtering rules restricted to what the flat model
    knows (collision_avoidance_limit.py:253-278): same-node (welded) geoms and parent/child
    nodes are skipped; ids ordered (min, max); duplicates kept as the reference keeps them."""
    def node_of(g):
        return fm.geom_frames[g].node

    out = []
    for ga, gb in groups:
        # the reference de-duplicates through list(set(ids)) (collision_avoidance_limit.py:246-247);
        # row order follows CPython's int-set iteration order, so do literally the same here.
        ia = list(set(names.index(n) if isinstance(n, str) else int(n) for n in ga))
        ib = list(set(names.index(n) if isinstance(n, str) else int(n) for n in gb))
        for a in ia:
            for b in ib:
                na, nb = node_of(a), node_of(b)
                if na == nb:
                    continue
                pa = fm.node_parent[na] if na >= 0 else -2
                pb = fm.node_parent[nb] if nb >= 0 else -2
                if pa == nb or pb == na:
                    continue
                if fm.geom_contype is not None and not ((fm.geom_contype[a] & fm.geom_conaffinity[b]) or
                                                        (fm.geom_contype[b] & fm.geom_conaffinity[a])):
                    continue   # contype / conaffinity filter (collision_avoidance_limit.py:269-278)
                out.append((min(a, b), max(a, b)))
    return out


def spec_from_workload(fm: FlatModel, wl: dict) -> ProblemSpec:
    tasks: List[TaskSpec] = []
    for f in wl["frames"]:
        cost = np.concatenate([np.broadcast_to(np.atleast_1d(f["position_cost"]).astype(float), 3),
                               np.broadcast_to(np.atleast_1d(f["orientation_cost"]).astype(float), 3)])
        tasks.append(TaskSpec(TASK_FRAME, frame=fm.frame(f["name"], f["type"]), cost=cost,
                              gain=f.get("gain", 1.0), lm_damping=f.get("lm_damping", 0.0)))
    for f in wl.get("relative_frames", []):
        cost = np.concatenate([np.broadcast_to(np.atleast_1d(f["position_cost"]).astype(float), 3),
                               np.broadcast_to(np.atleast_1d(f["orientation_cost"]).astype(float), 3)])
        tasks.append(TaskSpec(TASK_RELATIVE_FRAME, frame=fm.frame(f["name"], f["type"]), root=fm.frame(f["root_name"], f["root_type"]),
                              cost=cost, gain=f.get("gain", 1.0), lm_damping=f.get("lm_damping", 0.0)))
    if wl.get("posture") is not None:
        p = wl["posture"]
        tasks.append(TaskSpec(TASK_POSTURE, dof_cost=np.broadcast_to(np.atleast_1d(p["cost"]).astype(float), fm.nv).copy(),
                              gain=p.get("gain", 1.0), lm_damping=p.get("lm_damping", 0.0)))
    if wl.get("damping_task") is not None:   # DampingTask = PostureTask(gain 0, target qpos0), damping_task.py:19-20
        p = wl["damping_task"]
        tasks.append(TaskSpec(TASK_POSTURE, dof_cost=np.broadcast_to(np.atleast_1d(p["cost"]).astype(float), fm.nv).copy(),
                              gain=0.0, lm_damping=0.0))
    if wl.get("com") is not None:
        c = wl["com"]
        cost = np.zeros(6)
        cost[:3] = np.broadcast_to(np.atleast_1d(c["cost"]).astype(float), 3)
        tasks.append(TaskSpec(TASK_COM, cost=cost, gain=c.get("gain", 1.0), lm_damping=c.get("lm_damping", 0.0)))
    limits: List[LimitSpec] = []
    for l in wl["limits"]:
        if l["kind"] == "configuration":
            dof = np.nonzero(fm.dof_limited)[0].astype(np.int32)
            mind = l.get("min_distance_from_limits", 0.0)
            limits.append(LimitSpec(LIMIT_CONFIGURATION, dof=dof, lower=fm.dof_lo[dof] + mind,
                                    upper=fm.dof_hi[dof] - mind, gain=l.get("gain", 0.95)))
        elif l["kind"] == "velocity":
            dof = np.array([d for d in range(fm.nv) if fm.node_type[fm.dof_node[d]] != 0], dtype=np.int32)  # all but free joints
            limits.append(LimitSpec(LIMIT_VELOCITY, dof=dof, vmax=np.full(len(dof), float(l["vmax"]))))
        elif l["kind"] == "collision":
            names = fm.names["geom"]
            from .workloads import resolve_geom_groups

            id_pairs = _collision_pairs(fm, resolve_geom_groups(fm, l["pairs"]), names)
            used = sorted({g for p in id_pairs for g in p})
            local = {g: i for i, g in enumerate(used)}
            geoms = [(int(fm.geom_type[g]), fm.geom_frames[g], fm.geom_size[g]) for g in used]
            pairs = np.array([[local[a], local[b]] for a, b in id_pairs], dtype=np.int32).reshape(-1, 2)
            limits.append(LimitSpec(LIMIT_COLLISION, geoms=geoms, pairs=pairs, gain=l["gain"],
                                    minimum_distance=l["minimum_distance"],
                                    detection_distance=l["detection_distance"],
                                    bound_relaxation=l["bound_relaxation"]))
    return ProblemSpec(tasks, limits)
