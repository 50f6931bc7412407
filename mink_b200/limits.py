"""Kinematic limits with mink's interface (reference mink/limits/*.py).

`compute_qp_inequalities(configuration, dt)` returns `Constraint(G, h)` exactly as the reference lays
it out (G = [+P; -P], h = [upper; lower] for the box limits; one row per geom pair for collisions).
The numbers come from libbik (bik_limits_box / bik_fk_jac); only the constant +-projection G of the
box limits is assembled on the host.
"""

from __future__ import annotations

import abc
import itertools
from typing import Mapping, NamedTuple, Optional

import numpy as np

from ._abi import (LIMIT_COLLISION, LIMIT_CONFIGURATION, LIMIT_VELOCITY, LimitSpec, ProblemSpec)
from .configuration import Configuration, as_flat
from .exceptions import LimitDefinitionError

MJ_MAXVAL = 1e10


class Constraint(NamedTuple):
    """G(q) dq <= h(q); inactive when both are None (reference limits/limit.py:11-23)."""

    G: Optional[object] = None
    h: Optional[object] = None

    @property
    def inactive(self) -> bool:
        return self.G is None and self.h is None


class Limit(abc.ABC):
    @abc.abstractmethod
    def compute_qp_inequalities(self, configuration: Configuration, dt: float) -> Constraint:
        ...

    @abc.abstractmethod
    def _spec(self, flat) -> Optional[LimitSpec]:
        ...


def _box_constraint(limit: Limit, configuration: Configuration, dt: float, indices: np.ndarray) -> Constraint:
    from .tasks import problem_for

    prob = problem_for(configuration, ProblemSpec([], [limit._spec(configuration.flat)]))
    lo, hi = prob.box(configuration.q_device, dt)
    nv = configuration.nv
    P = np.eye(nv)[indices]
    G = np.vstack([P, -P])
    if configuration.batched:
        import torch

        idx = torch.as_tensor(np.array(indices), device=lo.device, dtype=torch.long)
        h = torch.cat([hi[:, idx], -lo[:, idx]], dim=1)
        return Constraint(torch.tensor(G, dtype=lo.dtype, device=lo.device).expand(lo.shape[0], -1, -1), h)
    ii = np.array(indices)
    h = np.concatenate([hi[0].cpu().numpy()[ii], -lo[0].cpu().numpy()[ii]]).astype(np.float64)
    return Constraint(G, h)


class ConfigurationLimit(Limit):
    """Joint position limits for slide/hinge joints; floating bases are ignored
    (reference limits/configuration_limit.py)."""

    def __init__(self, model, gain: float = 0.95, min_distance_from_limits: float = 0.0):
        if not 0.0 < gain <= 1.0:
            raise LimitDefinitionError(f"{self.__class__.__name__} gain must be in the range (0, 1]")
        flat = as_flat(model)
        lower = np.full(flat.nq, -MJ_MAXVAL)
        upper = np.full(flat.nq, MJ_MAXVAL)
        index_list = []
        for d in range(flat.nv):
            a = int(flat.dof_qadr[d])
            if a < 0 and flat.dof_limited[d] and int(flat.node_type[flat.dof_node[d]]) == 1:
                # the reference adds the three dofs of a limited ball joint (configuration_limit.py:44-56); the device box
                # has no cone limit, so refuse loudly instead of silently dropping the limit
                raise LimitDefinitionError(f"{self.__class__.__name__}: limited ball joints are not supported on the device "
                                           f"(joint {flat.names['joint'][int(flat.dof_node[d])]})")
            if a < 0 or not flat.dof_limited[d]:
                continue
            lower[a] = flat.dof_lo[d] + min_distance_from_limits
            upper[a] = flat.dof_hi[d] - min_distance_from_limits
            index_list.append(d)
        self.indices = np.array(index_list, dtype=np.int64)
        self.indices.setflags(write=False)
        self.projection_matrix = np.eye(flat.nv)[self.indices] if len(index_list) else None
        self.lower, self.upper = lower, upper     # read at call time, like the reference
        self.model, self.gain, self._flat = model, gain, flat

    def _spec(self, flat):
        if self.projection_matrix is None:
            return None
        qadr = flat.dof_qadr[self.indices]
        return LimitSpec(LIMIT_CONFIGURATION, dof=self.indices.astype(np.int32), lower=self.lower[qadr].copy(),
                         upper=self.upper[qadr].copy(), gain=self.gain)

    def compute_qp_inequalities(self, configuration: Configuration, dt: float) -> Constraint:
        """G = [P; -P], h = [gain (qmax - q); gain (q - qmin)] (configuration_limit.py:69-124)."""
        if self.projection_matrix is None:
            return Constraint()
        return _box_constraint(self, configuration, dt, self.indices)


class VelocityLimit(Limit):
    """|dq_i| <= dt vmax_i for the named joints (reference limits/velocity_limit.py)."""

    def __init__(self, model, velocities: Mapping[str, object] = {}):
        flat = as_flat(model)
        names = flat.names["joint"]
        limit_list, index_list = [], []
        for joint_name, max_vel in velocities.items():
            if joint_name not in names:
                raise KeyError(f"Invalid name '{joint_name}'. Valid names: {names}")
            jid = names.index(joint_name)
            jtype = int(flat.node_type[jid])
            if jtype == 0:
                raise LimitDefinitionError(f"Free joint {joint_name} is not supported")
            vadr, vdim = int(flat.node_dadr[jid]), (3 if jtype == 1 else 1)
            max_vel = np.atleast_1d(max_vel)
            if max_vel.shape != (vdim,):
                raise LimitDefinitionError(f"Joint {joint_name} must have a limit of shape ({vdim},). Got: {max_vel.shape}")
            index_list.extend(range(vadr, vadr + vdim))
            limit_list.extend(max_vel.tolist())
        self.indices = np.array(index_list, dtype=np.int64)
        self.indices.setflags(write=False)
        self.limit = np.array(limit_list, dtype=np.float64)
        self.limit.setflags(write=False)
        self.projection_matrix = np.eye(flat.nv)[self.indices] if len(index_list) else None

    def _spec(self, flat):
        if self.projection_matrix is None:
            return None
        return LimitSpec(LIMIT_VELOCITY, dof=self.indices.astype(np.int32), vmax=self.limit.copy())

    def compute_qp_inequalities(self, configuration: Configuration, dt: float) -> Constraint:
        """G = [P; -P], h = [dt vmax; dt vmax] (velocity_limit.py:71-101)."""
        if self.projection_matrix is None:
            return Constraint()
        return _box_constraint(self, configuration, dt, self.indices)


class CollisionAvoidanceLimit(Limit):
    """Normal-velocity limit between geom pairs (reference limits/collision_avoidance_limit.py).
    Supported geoms: plane, sphere, capsule, box (box against plane/sphere/capsule; SURVEY.md 7 hard part 6)."""

    def __init__(self, model, geom_pairs, gain: float = 0.85, minimum_distance_from_collisions: float = 0.005,
                 collision_detection_distance: float = 0.01, bound_relaxation: float = 0.0):
        self.model = model
        self._flat = as_flat(model)
        self.gain = gain
        self.minimum_distance_from_collisions = minimum_distance_from_collisions
        self.collision_detection_distance = collision_detection_distance
        self.bound_relaxation = bound_relaxation
        self.geom_id_pairs = self._construct_geom_id_pairs(geom_pairs)
        self.max_num_contacts = len(self.geom_id_pairs)

    def _construct_geom_id_pairs(self, geom_pairs):
        """Pair filtering of collision_avoidance_limit.py:253-278: geoms on the same weld group, on
        parent/child weld groups, or failing the contype/conaffinity test are skipped."""
        fm, names = self._flat, self._flat.names["geom"]

        def ids(group):
            return list(set(names.index(g) if isinstance(g, str) else int(g) for g in group))

        contype = getattr(self.model, "geom_contype", None)
        conaff = getattr(self.model, "geom_conaffinity", None)
        out = []
        for ga, gb in geom_pairs:
            for a, b in itertools.product(ids(ga), ids(gb)):
                na, nb = fm.geom_frames[a].node, fm.geom_frames[b].node
                if na == nb:
                    continue
                pa = fm.node_parent[na] if na >= 0 else -2
                pb = fm.node_parent[nb] if nb >= 0 else -2
                if pa == nb or pb == na:
                    continue
                if contype is not None and not ((contype[a] & conaff[b]) or (contype[b] & conaff[a])):
                    continue
                out.append((min(a, b), max(a, b)))
        return out

    def pair_mask(self, geoms) -> np.ndarray:
        """[len(geom_id_pairs)] bools: True for the pairs that involve any of `geoms` (names or ids).  For the per-instance
        `enabled` mask of solve_ik / converge_ik / track_ik's `collision` argument: ~limit.pair_mask(["wall"]) drops the wall."""
        names = self._flat.names["geom"]
        ids = set()
        for g in geoms:
            if isinstance(g, str):
                if g not in names:
                    raise LimitDefinitionError(f"pair_mask: no geom named {g!r}")
                ids.add(names.index(g))
            else:
                ids.add(int(g))
        return np.array([a in ids or b in ids for a, b in self.geom_id_pairs], dtype=bool)

    def _spec(self, flat):
        used = sorted({g for p in self.geom_id_pairs for g in p})
        local = {g: i for i, g in enumerate(used)}
        geoms = [(int(flat.geom_type[g]), flat.geom_frames[g], flat.geom_size[g]) for g in used]
        for t, _, _ in geoms:
            if t not in (0, 2, 3, 6):
                raise LimitDefinitionError("CollisionAvoidanceLimit: only plane, sphere, capsule and box geoms are supported on the device")
        for a, b in self.geom_id_pairs:
            if flat.geom_type[a] == 6 and flat.geom_type[b] == 6:
                raise LimitDefinitionError("CollisionAvoidanceLimit: box-box pairs are not supported on the device")
        pairs = np.array([[local[a], local[b]] for a, b in self.geom_id_pairs], dtype=np.int32).reshape(-1, 2)
        return LimitSpec(LIMIT_COLLISION, geoms=geoms, pairs=pairs, gain=self.gain,
                         minimum_distance=self.minimum_distance_from_collisions,
                         detection_distance=self.collision_detection_distance, bound_relaxation=self.bound_relaxation)

    def compute_qp_inequalities(self, configuration: Configuration, dt: float) -> Constraint:
        """Row = -n^T (Jp2 - Jp1); inactive rows are zero with h = +inf (collision_avoidance_limit.py:187-210)."""
        from .tasks import problem_for

        prob = problem_for(configuration, ProblemSpec([], [self._spec(configuration.flat)]))
        _, _, _, G, h = prob.fk_jac(configuration.q_device, dt=dt)
        if configuration.batched:
            return Constraint(G, h)
        return Constraint(G[0].cpu().numpy().astype(np.float64), h[0].cpu().numpy().astype(np.float64))
