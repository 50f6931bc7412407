"""build_ik / solve_ik with the reference signatures (mink/solve_ik.py:43-105) on the GPU engine.

`solve_ik` lowers the task and limit lists to ONE bik_problem (cached by layout) and issues one
bik_step: check_limits -> FK + Jacobians (K1) -> QP assembly + exact active-set solve (K2).
The `solver` string is accepted for drop-in compatibility and ignored: the device solver returns
the exact optimum of the same strictly convex QP that quadprog / daqp solve.
"""

from __future__ import annotations

from typing import NamedTuple, Optional, Sequence

import numpy as np

from ._abi import ProblemSpec
from .configuration import Configuration
from .exceptions import InvalidTarget, LimitDefinitionError, TargetNotSet
from .limits import CollisionAvoidanceLimit, ConfigurationLimit, Limit, VelocityLimit
from .tasks import ComTask, DampingTask, FrameTask, PostureTask, Task, problem_for


# status bits that fail a solve: BIK_STATUS_QP_MAXITER, _NONFINITE, _QP_INFEASIBLE, _BAD_WEIGHT
_QP_BITS = 2 | 4 | 8 | 32


class Problem(NamedTuple):
    """Stand-in for qpsolvers.Problem: min 1/2 x^T P x + q^T x  s.t.  G x <= h."""

    P: object
    q: object
    G: Optional[object]
    h: Optional[object]


def _problem(configuration: Configuration, tasks: Sequence[Task], limits: Optional[Sequence[Limit]]):
    flat = configuration.flat
    if limits is None:   # default of the reference (solve_ik.py:28-29)
        limits = [ConfigurationLimit(configuration.model)]
    tspecs = [t._spec(flat) for t in tasks]
    lspecs = [s for s in (l._spec(flat) for l in limits) if s is not None]
    return problem_for(configuration, ProblemSpec(tspecs, lspecs)), limits


def _posture_targets(tasks: Sequence[Task], nq: int, target=lambda t: t._target()):
    pt = [np.asarray(target(t)).reshape(-1, nq) for t in tasks if isinstance(t, PostureTask)]
    if not pt:
        return None
    nb = max(p.shape[0] for p in pt)
    return np.stack([np.broadcast_to(p, (nb, nq)) for p in pt], axis=1)


def _lower(configuration: Configuration, tasks: Sequence[Task], limits: Optional[Sequence[Limit]]):
    flat = configuration.flat
    prob, limits = _problem(configuration, tasks, limits)
    # libbik stacks rows by task kind order of appearance; keep frame / com targets in list order
    B = configuration.q_device.shape[0]
    ft = [np.broadcast_to(np.asarray(t._target()).reshape(-1, 7), (B, 7)) for t in tasks if isinstance(t, FrameTask)]
    pt = _posture_targets(tasks, flat.nq)
    ct = [np.broadcast_to(np.asarray(t._target()).reshape(-1, 3), (B, 3)) for t in tasks if isinstance(t, ComTask)]
    kw = {}
    if ft:
        kw["frame_targets"] = np.stack(ft, axis=1)
    if pt is not None:
        kw["posture_targets"] = pt
    if ct:
        kw["com_targets"] = np.stack(ct, axis=1)
    return prob, kw, limits


def _task_weights(tasks: Sequence[Task], weights, q, T: Optional[int] = None):
    """The [B, K] (track: [B, T, K]) weights buffer of a `weights={task: array}` mapping, rows in the stacked order of J
    (frame and CoM tasks in list order, 6 and 3 rows), 1 for tasks the mapping leaves out; None for no mapping.
    Per task: [k] or [B, k]; for a sequence (T given) [k], [T, k] or [B, T, k]."""
    if not weights:
        return None
    import torch

    for task in weights:
        if not isinstance(task, (FrameTask, ComTask)) or not any(task is t for t in tasks):
            raise InvalidTarget(f"weights apply to the FrameTask, RelativeFrameTask and ComTask of the task list, not {type(task).__name__}")
    B = q.shape[0]
    lead = (B,) if T is None else (B, T)
    blocks = []
    for task in tasks:
        if not isinstance(task, (FrameTask, ComTask)):
            continue
        k = 6 if isinstance(task, FrameTask) else 3
        w = weights.get(task)
        if w is None:
            blocks.append(torch.ones(lead + (k,), device=q.device, dtype=q.dtype))
            continue
        w = w if isinstance(w, torch.Tensor) else torch.as_tensor(np.array(w, dtype=np.float64))
        w = w.to(device=q.device, dtype=q.dtype)
        shapes = [(k,), (B, k)] if T is None else [(k,), (T, k), (B, T, k)]
        if tuple(w.shape) not in shapes:
            raise InvalidTarget(f"Expected weights of shape {' or '.join(str(list(s)) for s in shapes)} for {type(task).__name__}, got {list(w.shape)}")
        if T is not None and w.ndim == 2:
            w = w.unsqueeze(0)
        blocks.append(w.expand(lead + (k,)))
    return torch.cat(blocks, dim=-1).contiguous()


def _posture_weights(tasks: Sequence[Task], posture_weights, q, nv: int, T: Optional[int] = None):
    """The [B, P, nv] (track: [B, T, P, nv]) posture-weights buffer of a `posture_weights={task: w}` mapping, P the PostureTask /
    DampingTask of the task list in list order, 1 for those the mapping leaves out; None for no mapping.
    Per task: a float, [nv] or [B, nv]; for a sequence (T given) also [T, nv] or [B, T, nv]."""
    if not posture_weights:
        return None
    import torch

    for task in posture_weights:
        if not isinstance(task, PostureTask) or not any(task is t for t in tasks):
            raise InvalidTarget(f"posture_weights apply to the PostureTask and DampingTask of the task list, not {type(task).__name__}")
    B = q.shape[0]
    lead = (B,) if T is None else (B, T)
    blocks = []
    for task in tasks:
        if not isinstance(task, PostureTask):
            continue
        w = posture_weights.get(task)
        if w is None:
            blocks.append(torch.ones(lead + (nv,), device=q.device, dtype=q.dtype))
            continue
        w = w if isinstance(w, torch.Tensor) else torch.as_tensor(np.array(w, dtype=np.float64))
        w = w.to(device=q.device, dtype=q.dtype)
        shapes = [(), (nv,), (B, nv)] if T is None else [(), (nv,), (B, nv), (T, nv), (B, T, nv)]
        if tuple(w.shape) not in shapes:
            raise InvalidTarget(f"Expected posture weights of shape {' or '.join(str(list(s)) for s in shapes)} for {type(task).__name__}, "
                                f"got {list(w.shape)}")
        if T is not None and w.ndim == 2:
            if B == T and B > 1:
                raise InvalidTarget(f"posture weights of shape {list(w.shape)} could be [B, nv] or [T, nv] (B = T = {B}): pass [B, T, nv]")
            w = w.unsqueeze(1) if w.shape[0] == B else w.unsqueeze(0)
        blocks.append(w.expand(lead + (nv,)))
    return torch.stack(blocks, dim=-2).contiguous()


def _limit_bounds(limits: Optional[Sequence[Limit]], bounds, q, flat):
    """The (lower, upper, vmax) [B, nv] buffers of a `bounds={limit: value}` mapping, +-inf where nothing narrows; None for no
    mapping.  `limits` is the caller's list (None: the implicit default, which no key can name).
    ConfigurationLimit: (lower, upper), each None, [nq] or [B, nq] by qpos address; only the limit's listed dofs are read.
    VelocityLimit: vmax [k] or [B, k] in the order of limit.indices."""
    if not bounds:
        return None
    import torch

    B, nq, nv = q.shape[0], flat.nq, flat.nv
    listed = list(limits or [])
    full = lambda v: torch.full((B, nv), v, device=q.device, dtype=q.dtype)
    lo = up = vm = None

    def rows(x, n, what):
        x = x if isinstance(x, torch.Tensor) else torch.as_tensor(np.array(x, dtype=np.float64))
        x = x.to(device=q.device, dtype=q.dtype)
        if tuple(x.shape) not in ((n,), (B, n)):
            raise LimitDefinitionError(f"Expected {what} of shape [{n}] or [{B}, {n}], got {list(x.shape)}")
        return x.expand(B, n)

    for limit, value in bounds.items():
        if not isinstance(limit, (ConfigurationLimit, VelocityLimit)) or not any(limit is l for l in listed):
            raise LimitDefinitionError(f"bounds apply to the ConfigurationLimit and VelocityLimit of the limits list, not "
                                       f"{type(limit).__name__}" + (" (limits=None: the default ConfigurationLimit cannot be named)" if limits is None else ""))
        idx = torch.as_tensor(np.array(limit.indices), device=q.device, dtype=torch.long)
        if isinstance(limit, ConfigurationLimit):
            for other in listed:
                if other is not limit and isinstance(other, ConfigurationLimit) and np.intersect1d(other.indices, limit.indices).size:
                    raise LimitDefinitionError("bounds of a ConfigurationLimit that shares dofs with another ConfigurationLimit of the list "
                                               "are ambiguous: the device narrows every ConfigurationLimit of a dof")
            if not isinstance(value, (tuple, list)) or len(value) != 2:
                raise LimitDefinitionError("a ConfigurationLimit takes bounds (lower, upper), each None, [nq] or [B, nq]")
            qadr = torch.as_tensor(np.asarray(flat.dof_qadr)[np.asarray(limit.indices)], device=q.device, dtype=torch.long)
            if value[0] is not None:
                lo = full(-np.inf) if lo is None else lo
                lo[:, idx] = rows(value[0], nq, "lower bounds")[:, qadr]
            if value[1] is not None:
                up = full(np.inf) if up is None else up
                up[:, idx] = rows(value[1], nq, "upper bounds")[:, qadr]
        else:
            vm = full(np.inf) if vm is None else vm
            vm[:, idx] = torch.minimum(vm[:, idx], rows(value, len(limit.indices), "velocity caps"))
    return lo, up, vm


_COLLISION_KEYS = ("enabled", "minimum_distance_from_collisions", "collision_detection_distance")


def _collision(limits: Optional[Sequence[Limit]], collision, q, T: Optional[int] = None):
    """The (enabled, minimum_distance, detection_distance) buffers of a `collision={limit: {...}}` mapping, each None where the
    dict leaves the key out; None for no mapping.  enabled: bools over limit.geom_id_pairs, [npairs] or [B, npairs], for a
    sequence (T given) also [T, npairs] or [B, T, npairs]; the distances a float or [B], for a sequence also [T] or [B, T]."""
    if not collision:
        return None
    import torch

    listed = list(limits or [])
    if len(collision) != 1:
        raise LimitDefinitionError("collision takes one entry: the CollisionAvoidanceLimit of the limits list")
    (limit, value), = collision.items()
    if not isinstance(limit, CollisionAvoidanceLimit) or not any(limit is l for l in listed):
        raise LimitDefinitionError(f"collision applies to the CollisionAvoidanceLimit of the limits list, not {type(limit).__name__}")
    if not isinstance(value, dict) or not set(value) <= set(_COLLISION_KEYS):
        raise LimitDefinitionError(f"collision values are dicts with the keys {', '.join(_COLLISION_KEYS)}, each optional")
    B, npairs = q.shape[0], len(limit.geom_id_pairs)
    lead = (B,) if T is None else (B, T)

    def per_instance(x, tail, dtype, what):
        x = x if isinstance(x, torch.Tensor) else torch.as_tensor(np.array(x))
        x = x.to(device=q.device, dtype=dtype)
        shapes = [tail, (B,) + tail] if T is None else [tail, (B,) + tail, (T,) + tail, (B, T) + tail]
        if tuple(x.shape) not in shapes:
            raise LimitDefinitionError(f"Expected {what} of shape {' or '.join(str(list(s)) for s in shapes)}, got {list(x.shape)}")
        if T is not None and x.ndim == len(tail) + 1:
            if B == T and B > 1:
                raise LimitDefinitionError(f"{what} of shape {list(x.shape)} could be per instance or per frame (B = T = {B}): "
                                           f"pass {list((B, T) + tail)}")
            x = x.unsqueeze(1) if x.shape[0] == B else x.unsqueeze(0)
        return x.expand(lead + tail).contiguous()

    en = value.get("enabled")
    dmin = value.get("minimum_distance_from_collisions")
    ddet = value.get("collision_detection_distance")
    return (None if en is None else per_instance(np.asarray(en, dtype=bool) if not isinstance(en, torch.Tensor) else en != 0,
                                                 (npairs,), torch.uint8, "an enabled mask"),
            None if dmin is None else per_instance(dmin, (), q.dtype, "minimum_distance_from_collisions"),
            None if ddet is None else per_instance(ddet, (), q.dtype, "collision_detection_distance"))


def _frame_row(frame, dtype):
    """A frame's pose in its node as the problem image holds it (bik_build.h put_frame): the position, and the quaternion
    divided by its norm in double, then both in `dtype`."""
    import math

    q = [float(x) for x in frame.quat]
    n = math.sqrt(q[0] * q[0] + q[1] * q[1] + q[2] * q[2] + q[3] * q[3])
    n = n if n > 0 else 1.0
    return np.array([x / n for x in q] + [float(x) for x in frame.pos], dtype=np.float64).astype(dtype)


def _placement(tasks: Sequence[Task], placement, q, flat):
    """The [B, F, 7] placement buffer of a `placement={task: pose}` mapping, F the FrameTask / RelativeFrameTask of the task
    list in list order: each task's frame in its tree node, the problem's own for tasks the mapping leaves out; None for no
    mapping.  A pose is an SE3, a [7] or a [B, 7] array or tensor (wxyz_xyz) of the frame in its body, as model.site_pos /
    site_quat (geom_pos / geom_quat) hold it; it is composed with the body's pose in its node in fp64 as flatten composes a
    site (or geom), then stored in q's dtype as the problem image stores a frame."""
    if not placement:
        return None
    import torch

    for task in placement:
        if not isinstance(task, FrameTask) or not any(task is t for t in tasks):
            raise InvalidTarget(f"placement applies to the FrameTask and RelativeFrameTask of the task list, not {type(task).__name__}")
    B = q.shape[0]
    dt = np.float64 if q.dtype == torch.float64 else np.float32
    rows = []
    for task in tasks:
        if not isinstance(task, FrameTask):
            continue
        pose = placement.get(task)
        if pose is None:
            rows.append(np.broadcast_to(_frame_row(task._spec(flat).frame, dt), (B, 7)))
            continue
        if hasattr(pose, "wxyz_xyz"):
            pose = pose.wxyz_xyz
        p = pose.detach().cpu().numpy() if isinstance(pose, torch.Tensor) else np.asarray(pose)
        p = p.astype(np.float64)
        if p.shape not in ((7,), (B, 7)):
            raise InvalidTarget(f"Expected a placement of shape [7] or [{B}, 7] for {type(task).__name__}, got {list(p.shape)}")
        try:
            flat.frame_body(task.frame_name, task.frame_type)
        except (KeyError, ValueError) as e:
            raise InvalidTarget(f"cannot place the frame of {type(task).__name__} {task.frame_name!r}: {e}") from None
        p = p.reshape(-1, 7)
        uniq, inv = np.unique(p, axis=0, return_inverse=True)   # the composition is per distinct pose
        placed = np.stack([_frame_row(flat.placed_frame(task.frame_name, task.frame_type, u[4:], u[:4]), dt) for u in uniq])
        rows.append(np.broadcast_to(placed[inv.reshape(-1)], (B, 7)))
    return torch.as_tensor(np.ascontiguousarray(np.stack(rows, axis=1)), device=q.device)


def build_ik(configuration: Configuration, tasks: Sequence[Task], dt: float, damping: float = 1e-12,
             limits: Optional[Sequence[Limit]] = None) -> Problem:
    """QP of the IK problem (reference solve_ik.py:43-65): P = damping I + sum H_t, q = sum c_t,
    G / h stacked over the limits in list order (None when there is no inequality)."""
    prob, kw, limits = _lower(configuration, tasks, limits)
    J, e, ep, _, _ = prob.fk_jac(configuration.q_device, dt=dt, **kw)
    H, c = prob.objective(J, e, ep, damping)
    G_list, h_list = [], []
    for limit in limits:
        con = limit.compute_qp_inequalities(configuration, dt)
        if not con.inactive:
            G_list.append(con.G)
            h_list.append(con.h)
    if configuration.batched:
        import torch

        G = torch.cat([g.to(h_list[0].dtype) for g in G_list], dim=1) if G_list else None
        h = torch.cat(list(h_list), dim=1) if h_list else None
        return Problem(H, c, G, h)
    G = np.vstack(G_list) if G_list else None
    h = np.hstack(h_list) if h_list else None
    return Problem(H[0].cpu().numpy(), c[0].cpu().numpy(), G, h)


def solve_ik(configuration: Configuration, tasks: Sequence[Task], dt: float, solver: str = "b200", damping: float = 1e-12,
             safety_break: bool = False, limits: Optional[Sequence[Limit]] = None, weights=None, posture_weights=None, bounds=None,
             collision=None, placement=None, **kwargs):
    """Velocity v = dq / dt tangent to the configuration (reference solve_ik.py:68-105).

    `weights` maps a FrameTask / RelativeFrameTask to a [6] or [B, 6] array and a ComTask to a [3] or [B, 3] array of
    multipliers in [0, 1] of the task's costs (position xyz, orientation xyz): instance b solves with cost * w[b], as if the
    task's costs had been set to that.  Tasks missing from the mapping keep their costs.

    `posture_weights` maps a PostureTask / DampingTask to a float, an [nv] or a [B, nv] array of multipliers in [0, 1] of the
    task's per-dof costs: instance b solves as if the task's cost had been set to cost * w[b] (PostureTask.set_cost).  A
    weight of 0 on every dof of a DampingTask solves that instance as if the task were not in the list.

    `bounds` maps a ConfigurationLimit of `limits` to (lower, upper), each None, [nq] or [B, nq] indexed by qpos address like
    ConfigurationLimit.lower / upper, and a VelocityLimit of `limits` to vmax, [k] or [B, k] in the order of its indices like
    VelocityLimit.limit.  They narrow the limit's bounds per instance: instance b solves as if the limit had been built with
    max(lower, lower[b]), min(upper, upper[b]) and min(vmax, vmax[b]) on the dofs it lists; other entries are not read.  The
    values are final bounds (any min_distance_from_limits margin is the caller's to apply), they can only narrow, and a
    ConfigurationLimit that shares dofs with another one of the list cannot be a key.  A cap of 0 keeps a dof where it is.
    build_ik and compute_qp_inequalities still show the limits' own bounds.

    `collision` maps the CollisionAvoidanceLimit of `limits` to a dict with any of the keys "enabled",
    "minimum_distance_from_collisions" and "collision_detection_distance".  "enabled" is a bool array over the limit's
    geom_id_pairs, [npairs] or [B, npairs]: instance b solves as if the limit had been built with its enabled pairs only
    (limit.pair_mask(geoms) selects the pairs that involve some geoms).  The distances are a float or a [B] array that
    replace the limit's attributes of those names per instance; a non-finite distance keeps the limit's own and flags the
    instance.  compute_qp_inequalities still shows the limit's own pairs and distances.

    `placement` maps a FrameTask / RelativeFrameTask of `tasks` to the pose of its frame in its body, an SE3 or a [7] or
    [B, 7] array (wxyz_xyz): what model.site_pos / site_quat (geom_pos / geom_quat) hold for a site (geom) frame, a pose in
    the body for a body frame (identity: the body itself).  Instance b solves as if the model had been built with its
    frame there: one marker placement per performer, one tool length per instance, one contact point per grasp.  A
    RelativeFrameTask's root keeps its place, and tasks left out keep the model's.  Task.compute_error / compute_jacobian
    still use the model's placement.

    Returns a numpy (nv,) vector for a single configuration, a torch CUDA [B, nv] tensor for a batch.
    Raises NotWithinConfigurationLimits when `safety_break` and some instance is out of limits;
    raises AssertionError (like the reference's `assert dq is not None`) when the QP of any instance
    could not be solved.
    """
    limits_arg = limits   # the caller's list: `bounds` and `collision` keys name its limits
    prob, kw, limits = _lower(configuration, tasks, limits)
    q = configuration.q_device
    w = _task_weights(tasks, weights, q)
    pw = _posture_weights(tasks, posture_weights, q, configuration.flat.nv)
    bd = _limit_bounds(limits_arg, bounds, q, configuration.flat)
    co = _collision(limits_arg, collision, q)
    pl = _placement(tasks, placement, q, configuration.flat)
    dq, status = prob.step(q, dt=dt, damping=damping, nsteps=1, integrate=False, weights=w, posture_weights=pw, bounds=bd, collision=co,
                           placement=pl, **kw)
    st = status.cpu().numpy()
    if (st & 1).any():
        if safety_break:
            configuration.check_limits(safety_break=True)
        else:
            configuration.check_limits(safety_break=False)
    assert not (st & _QP_BITS).any(), f"QP not solved for {int(((st & _QP_BITS) != 0).sum())} instance(s) (status bits {np.unique(st & _QP_BITS)})"
    v = dq / float(dt)
    if configuration.batched:
        return v
    return v[0].cpu().numpy().astype(np.float64)


def converge_ik(configuration: Configuration, tasks: Sequence[Task], dt: float, solver: str = "b200", damping: float = 1e-12,
                limits: Optional[Sequence[Limit]] = None, max_iters: int = 20, pos_threshold: float = 1e-4,
                ori_threshold: float = 1e-4, check_every: int = 1, weights=None, posture_weights=None, bounds=None, collision=None,
                placement=None):
    """The inner loop the reference's examples wrap around solve_ik (examples/arm_iiwa.py:63-70,
    examples/quadruped_spot.py:89-104), run on the device per instance:

        for i in range(max_iters):
            vel = solve_ik(configuration, tasks, dt, solver, damping, limits=limits)
            configuration.integrate_inplace(vel, dt)
            if every FrameTask/RelativeFrameTask: |err[:3]| <= pos_threshold and |err[3:]| <= ori_threshold: break

    The configuration is updated in place; returns (iters, converged): steps taken and whether the thresholds were
    met, numpy scalars for a single configuration, [B] numpy arrays for a batch.  A single configuration and a float64
    batch run in fp64 end to end (bik_converge64), a float32 batch on the fp32 fast path.

    `weights` as in solve_ik.  A frame task whose three position (orientation) weights are 0 in an instance is left out of
    that instance's position (orientation) test.  `posture_weights`, `bounds`, `collision` and `placement` as in solve_ik;
    the thresholds are tested on the placed frames' errors."""
    limits_arg = limits   # the caller's list: `bounds` and `collision` keys name its limits
    prob, kw, limits = _lower(configuration, tasks, limits)
    q = configuration.q_device
    w = _task_weights(tasks, weights, q)
    pw = _posture_weights(tasks, posture_weights, q, configuration.flat.nv)
    bd = _limit_bounds(limits_arg, bounds, q, configuration.flat)
    co = _collision(limits_arg, collision, q)
    pl = _placement(tasks, placement, q, configuration.flat)
    iters, status = prob.converge(q, dt=dt, damping=damping, max_iters=max_iters, pos_threshold=pos_threshold,
                                  ori_threshold=ori_threshold, check_every=check_every, weights=w, posture_weights=pw, bounds=bd,
                                  collision=co, placement=pl, **kw)
    configuration._sync_from_device()
    st = status.cpu().numpy()
    assert not (st & _QP_BITS).any(), f"QP not solved for {int(((st & _QP_BITS) != 0).sum())} instance(s) (status bits {np.unique(st & _QP_BITS)})"
    it, ok = iters.cpu().numpy(), (st & 16) == 0
    if configuration.batched:
        return it, ok
    return int(it[0]), bool(ok[0])


def track_ik(configuration: Configuration, tasks: Sequence[Task], dt: float, targets, solver: str = "b200",
             damping: float = 1e-12, limits: Optional[Sequence[Limit]] = None, max_iters: int = 20, pos_threshold: float = 1e-4,
             ori_threshold: float = 1e-4, lengths=None, check_every: int = 1, weights=None, posture_weights=None, bounds=None,
             collision=None, hold=None, placement=None):
    """The examples' outer loop (examples/arm_aloha.py:140-169) over a sequence of targets, run on the device:

        for t in range(T):
            for task, seq in targets.items(): task.set_target(seq[t])
            converge_ik(configuration, tasks, dt, solver, damping, limits, max_iters, pos_threshold, ori_threshold)

    with every instance of a batch moving to its next frame as soon as it is done with the current one.

    `targets` maps a FrameTask / RelativeFrameTask to its [T, 7] or [B, T, 7] sequence (an SE3 or an array / tensor,
    wxyz_xyz) and a ComTask to its [T, 3] or [B, T, 3] sequence; a sequence without a batch dimension is shared by every
    instance, and a task not in `targets` keeps its current target.  CUDA tensors are used where they are.  `lengths`
    ([B], each in 0..T) ends instance b's sequence after lengths[b] frames.  The configuration ends at its final q.

    Sequences take the configuration's precision: a single configuration and a float64 batch run in fp64 end to end
    (bik_track64), a float32 batch on the fp32 fast path.

    A PostureTask takes a [T, nq] or [B, T, nq] sequence of joint-space targets in `targets` as well (a retargeted source
    motion, say); posture tasks not in `targets` keep their current target on every frame.  A DampingTask's target is qpos0,
    so it takes no sequence.

    `weights` as in converge_ik, per frame: a task's weights are [6] / [3] (every frame), [T, 6] / [T, 3] (shared by every
    instance) or [B, T, 6] / [B, T, 3].  Posture tasks have no `weights`.

    `posture_weights` as in converge_ik, per frame: a PostureTask's or DampingTask's weights are a float, [nv] or [B, nv]
    (every frame), [T, nv] (shared by every instance) or [B, T, nv] (a 2-D array must then not leave B = T ambiguous).

    `bounds` as in solve_ik, one value per instance that holds on every frame.

    `collision` as in solve_ik, per frame: "enabled" is [npairs] or [B, npairs] (every frame), [T, npairs] (shared by every
    instance) or [B, T, npairs]; a distance is a float or [B] (every frame), [T] or [B, T] (a 2-D mask or a 1-D distance must
    then not leave B = T ambiguous).

    `hold` maps a FrameTask, RelativeFrameTask, ComTask or PostureTask to a [T] or [B, T] mask of the frames it is held on.
    Over each run of consecutive held frames the task's target is its value at the configuration the run begins from, as if
    task.set_target_from_configuration(configuration) were called before the run's first frame: contact locking, a foot held
    where it touched down for as long as the contact lasts.  The value is captured on the device; it replaces the task's
    sequence or target on the held frames.  A task held on every frame of every instance needs neither a sequence nor a
    target.  A DampingTask cannot be held.

    `placement` as in solve_ik, one pose per instance that holds on every frame (a performer's markers, a tool).  A held
    FrameTask captures the world pose of its placed frame, a held RelativeFrameTask that frame's pose in its root.

    Returns (q_traj, iters, converged) per frame: numpy float64 [T, nq] / [T] / [T] for a single configuration, torch
    CUDA [B, T, nq] (q's dtype) / [B, T] / [B, T] for a batch (rows past an instance's length: NaN, -1, False)."""
    import torch

    for task in targets:
        if not isinstance(task, (FrameTask, ComTask, PostureTask)) or isinstance(task, DampingTask):
            raise InvalidTarget(f"track_ik takes target sequences for FrameTask, RelativeFrameTask, ComTask and PostureTask, "
                                f"not {type(task).__name__}")
    hold = hold or {}
    for task in hold:
        if not isinstance(task, (FrameTask, ComTask, PostureTask)) or isinstance(task, DampingTask) or task not in tasks:
            raise InvalidTarget(f"track_ik holds FrameTask, RelativeFrameTask, ComTask and PostureTask targets of `tasks`, "
                                f"not {type(task).__name__}")
    flat = configuration.flat
    q = configuration.q_device
    B, dev = q.shape[0], q.device
    masks = {}
    for task, m in hold.items():
        m = (m if isinstance(m, torch.Tensor) else torch.as_tensor(np.asarray(m))).to(device=dev) != 0
        if m.ndim == 1:
            m = m.unsqueeze(0).expand(B, -1)
        if m.ndim != 2 or m.shape[0] != B or m.shape[1] < 1:
            raise InvalidTarget(f"Expected a [T] or [{B}, T] hold mask for {type(task).__name__}, got {tuple(m.shape)}")
        masks[task] = m
    always = {t for t, m in masks.items() if bool(m.all())}   # held on every frame: its target rows are ignored

    def target_of(t, fill):
        try:
            return np.asarray(t._target(), dtype=np.float64)
        except TargetNotSet:
            if t not in always:
                raise
            return np.asarray(fill, dtype=np.float64)

    fills = {FrameTask: [1, 0, 0, 0, 0, 0, 0], ComTask: [0, 0, 0], PostureTask: np.asarray(flat.qpos0, dtype=np.float64)}
    fill_of = lambda t: next(v for k, v in fills.items() if isinstance(t, k))
    for t in tasks:
        if isinstance(t, (FrameTask, ComTask)) and t not in targets:
            target_of(t, fill_of(t))   # TargetNotSet when a task has neither a sequence nor a target (nor is always held)
    seqs, T = {}, None
    for task, seq in targets.items():
        k = 7 if isinstance(task, FrameTask) else (flat.nq if isinstance(task, PostureTask) else 3)
        if hasattr(seq, "wxyz_xyz"):
            seq = seq.wxyz_xyz
        s = seq if isinstance(seq, torch.Tensor) else torch.as_tensor(np.asarray(seq, dtype=np.float64))
        s = s.to(device=dev, dtype=q.dtype)
        if s.ndim == 2:
            s = s.unsqueeze(0).expand(B, -1, -1)
        if s.ndim != 3 or s.shape[0] != B or s.shape[2] != k or s.shape[1] < 1:
            raise InvalidTarget(f"Expected a [T, {k}] or [{B}, T, {k}] target sequence for {type(task).__name__}, got {tuple(s.shape)}")
        if T is not None and s.shape[1] != T:
            raise InvalidTarget(f"target sequences of different lengths: {T} and {s.shape[1]} frames")
        T = s.shape[1]
        seqs[task] = s
    for task, m in masks.items():
        if T is not None and m.shape[1] != T:
            raise InvalidTarget(f"the hold mask of {type(task).__name__} has {m.shape[1]} frames, the sequences {T}")
        T = m.shape[1]
    if T is None:
        raise InvalidTarget("track_ik needs at least one FrameTask / RelativeFrameTask / ComTask / PostureTask target sequence")

    def stacked(kind, k):
        rows = [seqs[t] if t in seqs else torch.as_tensor(target_of(t, fill_of(t)).reshape(-1, 1, k), device=dev,
                                                          dtype=q.dtype).expand(B, T, k)
                for t in tasks if isinstance(t, kind)]
        return torch.stack(rows, dim=2).contiguous() if rows else None

    posture, posture_seq = _posture_targets(tasks, flat.nq, lambda t: target_of(t, fill_of(t))), False
    if any(isinstance(t, PostureTask) for t in seqs):
        # one [1 or B, T, nq] block per posture task (a sequence given without a batch dimension, or a held target shared by
        # the batch: 1); [T, P, nq] when every block is shared, else [B, T, P, nq]
        rows = [(seqs[t][:1] if seqs[t].stride(0) == 0 else seqs[t]) if t in seqs else
                torch.as_tensor(target_of(t, fill_of(t)).reshape(-1, 1, flat.nq), device=dev, dtype=q.dtype).expand(-1, T, -1)
                for t in tasks if isinstance(t, PostureTask)]
        lead = max(r.shape[0] for r in rows)
        posture = torch.stack([r.expand(lead, T, flat.nq) for r in rows], dim=2).contiguous()
        posture, posture_seq = (posture[0] if lead == 1 else posture), True

    limits_arg = limits   # the caller's list: `bounds` and `collision` keys name its limits
    prob, limits = _problem(configuration, tasks, limits)
    w = _task_weights(tasks, weights, q, T)
    pw = _posture_weights(tasks, posture_weights, q, flat.nv, T)
    bd = _limit_bounds(limits_arg, bounds, q, flat)
    co = _collision(limits_arg, collision, q, T)
    pl = _placement(tasks, placement, q, flat)
    ln = None
    if lengths is not None:
        ln = lengths.to(device=dev, dtype=torch.int32) if isinstance(lengths, torch.Tensor) else torch.as_tensor(np.asarray(lengths, dtype=np.int32), device=dev)
        if ln.shape != (B,):
            raise InvalidTarget(f"lengths must have shape ({B},), got {tuple(ln.shape)}")
    hd = None
    if masks:   # columns: frame-like tasks, CoM tasks, posture-type tasks, each in the order of `tasks`, as the targets are stacked
        cols = [t for t in tasks if isinstance(t, FrameTask)] + [t for t in tasks if isinstance(t, ComTask)] + \
               [t for t in tasks if isinstance(t, PostureTask)]
        hd = torch.zeros((B, T, len(cols)), device=dev, dtype=torch.uint8)
        for k, t in enumerate(cols):
            if t in masks:
                hd[:, :, k] = masks[t].to(torch.uint8)
    q_traj, iters, status, _ = prob.track(q, stacked(FrameTask, 7), posture, stacked(ComTask, 3), lengths=ln, dt=dt,
                                          damping=damping, max_iters=max_iters, pos_threshold=pos_threshold,
                                          ori_threshold=ori_threshold, check_every=check_every, weights=w, posture_seq=posture_seq,
                                          posture_weights=pw, bounds=bd, collision=co, hold=hd, placement=pl)
    configuration._sync_from_device()
    ran = iters >= 0
    bad = ((status & _QP_BITS) != 0) & ran
    n_bad = int(bad.sum())
    assert n_bad == 0, f"QP not solved for {n_bad} frame(s) (status bits {np.unique((status[bad] & _QP_BITS).cpu().numpy())})"
    converged = ran & ((status & 16) == 0)
    if configuration.batched:
        return q_traj, iters, converged
    return q_traj[0].cpu().numpy(), iters[0].cpu().numpy(), converged[0].cpu().numpy()
