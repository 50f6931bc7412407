"""Flatten an MjModel-shaped model into the kinematic-tree blob consumed by libbik.

The hot path never sees MuJoCo structures.  At setup time the front end reduces the model to
a list of *nodes* -- one per joint, parents first -- with the static transform from the parent
node, the joint axis/anchor in the node frame and the qpos/dof addresses (BASELINE.json
north_star: "a flattened kinematic tree (joint types, parent indices, local SE(3) offsets)").
Bodies without joints are folded into the offset of whatever hangs below them, so FK on the
device walks `njnt` nodes instead of `nbody` bodies (G1: 38 instead of 44).

Replaces what the reference reads per step out of MjModel inside mj_kinematics / mj_jac
(reference mink/configuration.py:63-64,144-145; semantics SURVEY.md A.2).

Blob layout (little endian), shared with include/bik.h and oracle/ik_oracle.c:
  header  : u32 magic 'BIKM', u32 version, u32 nbytes, u32 nsections,
            i32 nq, nv, nnode, ncom, 4 x i32 reserved                      (48 bytes)
  table   : nsections x { char name[20]; u32 dtype (0=i32, 1=f64); u32 count; u32 offset }
  payload : 16-byte aligned arrays
"""

from __future__ import annotations

import json
import struct
from dataclasses import dataclass, field
from typing import Dict, List

import numpy as np

from .mjcf import DOF_WIDTH, JNT_BALL, JNT_FREE, JNT_HINGE, JNT_SLIDE, QPOS_WIDTH  # noqa: F401  (re-exported through __all__)

BLOB_MAGIC = 0x4D4B4942  # 'BIKM'
BLOB_VERSION = 1
_HDR = struct.Struct("<4I8i")
_SEC = struct.Struct("<20s3I")


def _qmul(a, b):
    return np.array([
        a[0] * b[0] - a[1] * b[1] - a[2] * b[2] - a[3] * b[3],
        a[0] * b[1] + a[1] * b[0] + a[2] * b[3] - a[3] * b[2],
        a[0] * b[2] - a[1] * b[3] + a[2] * b[0] + a[3] * b[1],
        a[0] * b[3] + a[1] * b[2] - a[2] * b[1] + a[3] * b[0],
    ])


def _qrot(q, v):
    w, x, y, z = q
    R = np.array([
        [1 - 2 * (y * y + z * z), 2 * (x * y - w * z), 2 * (x * z + w * y)],
        [2 * (x * y + w * z), 1 - 2 * (x * x + z * z), 2 * (y * z - w * x)],
        [2 * (x * z - w * y), 2 * (y * z + w * x), 1 - 2 * (x * x + y * y)],
    ])
    return R @ v


def _compose(p1, q1, p2, q2):
    q = _qmul(q1, q2)
    return p1 + _qrot(q1, p2), q / np.linalg.norm(q)


@dataclass
class Frame:
    """A frame rigidly attached to a node (-1 = fixed in the world)."""

    node: int
    pos: np.ndarray
    quat: np.ndarray


@dataclass
class FlatModel:
    nq: int
    nv: int
    nnode: int
    node_parent: np.ndarray   # i32 [nnode]   parent node, -1 = world
    node_type: np.ndarray     # i32 [nnode]   mjtJoint code (0 free, 1 ball, 2 slide, 3 hinge)
    node_qadr: np.ndarray     # i32 [nnode]
    node_dadr: np.ndarray     # i32 [nnode]
    node_pos: np.ndarray      # f64 [nnode,3] offset parent-node frame -> this node (pre-joint)
    node_quat: np.ndarray     # f64 [nnode,4]
    node_axis: np.ndarray     # f64 [nnode,3] joint axis in the node frame (unit)
    node_jpos: np.ndarray     # f64 [nnode,3] joint anchor in the node frame
    qpos0: np.ndarray         # f64 [nq]
    dof_node: np.ndarray      # i32 [nv]
    dof_qadr: np.ndarray      # i32 [nv]      qpos index for slide/hinge dofs, -1 for free/ball dofs
    dof_limited: np.ndarray   # i32 [nv]
    dof_lo: np.ndarray        # f64 [nv]      joint range (only meaningful where dof_limited)
    dof_hi: np.ndarray        # f64 [nv]
    com_node: np.ndarray      # i32 [ncom]    node carrying each massive body of subtree(body 1)
    com_pos: np.ndarray       # f64 [ncom,3]  inertial-frame origin in that node's frame
    com_mass: np.ndarray      # f64 [ncom]
    # host-side bookkeeping (not in the blob)
    body_frames: List[Frame] = field(default_factory=list)   # every MuJoCo body as (node, offset)
    names: Dict[str, list] = field(default_factory=dict)
    site_frames: List[Frame] = field(default_factory=list)
    geom_frames: List[Frame] = field(default_factory=list)
    key_qpos: np.ndarray = None
    com_missing: list = None   # bodies of subtree(body 1) whose mass the MJCF compiler could not derive (no <inertial>)
    geom_type: np.ndarray = None
    body_parentid: np.ndarray = None      # MJCF body tree and geom -> body map: what mink_b200.utils walks; None: not recorded
    geom_bodyid: np.ndarray = None
    site_bodyid: np.ndarray = None        # site -> body map: where a site sits (placement of a site frame); None: not recorded
    geom_contype: np.ndarray = None       # collision filter bits (collision_avoidance_limit.py:269-278); None: not recorded
    geom_conaffinity: np.ndarray = None
    geom_size: np.ndarray = None
    jnt_limited: np.ndarray = None
    jnt_range: np.ndarray = None

    @property
    def ncom(self) -> int:
        return int(self.com_mass.shape[0])

    # ---- frame lookup ------------------------------------------------------ #
    def frame(self, name: str, kind: str) -> Frame:
        """(node, offset) of a named body / geom / site (reference configuration.py:133,170)."""
        table = {"body": self.body_frames, "geom": self.geom_frames, "site": self.site_frames}[kind]
        names = self.names[kind]
        if name not in names:
            raise KeyError(name)
        return table[names.index(name)]

    def frame_body(self, name: str, kind: str) -> int:
        """MuJoCo body a named body / geom / site frame is fixed to.  ValueError when the model does not record it (a site
        of a model whose metadata predates site_bodyid)."""
        i = self.names[kind].index(name)
        if kind == "body":
            return i
        ids = self.site_bodyid if kind == "site" else self.geom_bodyid
        if ids is None:
            raise ValueError(f"the model does not record which body each {kind} belongs to")
        return int(ids[i])

    def placed_frame(self, name: str, kind: str, pos, quat) -> Frame:
        """The frame `name` of `kind` placed at pose (pos, quat) in its body: what flatten gives the frame of a model whose
        site_pos / site_quat (geom_pos / geom_quat) hold that pose, composed as flatten's attach composes it.  For a body, a
        pose in that body (identity: the body itself)."""
        f = self.body_frames[self.frame_body(name, kind)]
        p, q = _compose(f.pos, f.quat, np.asarray(pos, dtype=np.float64), np.asarray(quat, dtype=np.float64))
        return Frame(f.node, p, q)

    # ---- blob -------------------------------------------------------------- #
    _SECTIONS = ("node_parent", "node_type", "node_qadr", "node_dadr", "node_pos", "node_quat",
                 "node_axis", "node_jpos", "qpos0", "dof_node", "dof_qadr", "dof_limited",
                 "dof_lo", "dof_hi", "com_node", "com_pos", "com_mass")

    def to_blob(self) -> bytes:
        arrays = []
        for name in self._SECTIONS:
            a = np.ascontiguousarray(getattr(self, name))
            if a.dtype.kind in "iub":
                a = a.astype("<i4")
                code = 0
            else:
                a = a.astype("<f8")
                code = 1
            arrays.append((name, code, a))
        table_bytes = _SEC.size * len(arrays)
        off = _HDR.size + table_bytes
        off = (off + 15) & ~15
        entries, payload = [], bytearray()
        for name, code, a in arrays:
            raw = a.tobytes()
            entries.append(_SEC.pack(name.encode(), code, a.size, off + len(payload)))
            payload += raw
            payload += b"\0" * ((-len(payload)) % 16)
        nbytes = off + len(payload)
        hdr = _HDR.pack(BLOB_MAGIC, BLOB_VERSION, nbytes, len(arrays),
                        self.nq, self.nv, self.nnode, self.ncom, 0, 0, 0, 0)
        head = hdr + b"".join(entries)
        head += b"\0" * (off - len(head))
        return bytes(head + payload)

    def to_meta_json(self) -> str:
        """Names + frame tables + keyframes, so fixtures can be used without the MJCF."""
        def fr(fs):
            return [[int(f.node)] + [float(x) for x in f.pos] + [float(x) for x in f.quat] for f in fs]
        return json.dumps(dict(
            names=self.names, body_frames=fr(self.body_frames), site_frames=fr(self.site_frames),
            geom_frames=fr(self.geom_frames), key_qpos=self.key_qpos.tolist(),
            geom_type=self.geom_type.tolist(), geom_size=self.geom_size.tolist(),
            jnt_limited=[int(x) for x in self.jnt_limited], jnt_range=self.jnt_range.tolist(),
            com_missing=list(self.com_missing or []),
            body_parentid=None if self.body_parentid is None else [int(x) for x in self.body_parentid],
            geom_bodyid=None if self.geom_bodyid is None else [int(x) for x in self.geom_bodyid],
            site_bodyid=None if self.site_bodyid is None else [int(x) for x in self.site_bodyid],
            geom_contype=None if self.geom_contype is None else [int(x) for x in self.geom_contype],
            geom_conaffinity=None if self.geom_conaffinity is None else [int(x) for x in self.geom_conaffinity]))

    @classmethod
    def from_blob(cls, blob: bytes, meta_json: str = None) -> "FlatModel":
        magic, version, nbytes, nsec, nq, nv, nnode, ncom, *_ = _HDR.unpack_from(blob, 0)
        if magic != BLOB_MAGIC or version != BLOB_VERSION or nbytes != len(blob):
            raise ValueError("not a BIKM v1 blob")
        kw = {}
        for s in range(nsec):
            name, code, count, off = _SEC.unpack_from(blob, _HDR.size + s * _SEC.size)
            name = name.rstrip(b"\0").decode()
            a = np.frombuffer(blob, dtype="<i4" if code == 0 else "<f8", count=count, offset=off).copy()
            kw[name] = a
        for k, w in (("node_pos", 3), ("node_quat", 4), ("node_axis", 3), ("node_jpos", 3), ("com_pos", 3)):
            kw[k] = kw[k].reshape(-1, w)
        fm = cls(nq=nq, nv=nv, nnode=nnode, **kw)
        if meta_json is not None:
            meta = json.loads(meta_json)
            def fr(rows):
                return [Frame(int(r[0]), np.array(r[1:4]), np.array(r[4:8])) for r in rows]
            fm.names = meta["names"]
            fm.body_frames = fr(meta["body_frames"])
            fm.site_frames = fr(meta["site_frames"])
            fm.geom_frames = fr(meta["geom_frames"])
            fm.key_qpos = np.array(meta["key_qpos"]).reshape(-1, nq)
            fm.com_missing = list(meta.get("com_missing", []))
            fm.geom_type = np.array(meta["geom_type"], dtype=np.int32)
            fm.geom_size = np.array(meta["geom_size"]).reshape(-1, 3)
            fm.jnt_limited = np.array(meta["jnt_limited"], dtype=bool)
            fm.jnt_range = np.array(meta["jnt_range"]).reshape(-1, 2)
            if meta.get("body_parentid") is not None:
                fm.body_parentid = np.array(meta["body_parentid"], dtype=np.int32)
                fm.geom_bodyid = np.array(meta["geom_bodyid"], dtype=np.int32)
            if meta.get("site_bodyid") is not None:
                fm.site_bodyid = np.array(meta["site_bodyid"], dtype=np.int32)
            if meta.get("geom_contype") is not None:
                fm.geom_contype = np.array(meta["geom_contype"], dtype=np.int32)
                fm.geom_conaffinity = np.array(meta["geom_conaffinity"], dtype=np.int32)
        return fm

    # what mink_b200.utils needs of an MjModel (geoms of one body are contiguous in MuJoCo's tables)
    @property
    def nbody(self) -> int:
        return len(self.body_parentid)

    @property
    def body_geomnum(self) -> np.ndarray:
        return np.bincount(self.geom_bodyid, minlength=self.nbody).astype(np.int32)

    @property
    def body_geomadr(self) -> np.ndarray:
        num = self.body_geomnum
        first = np.full(self.nbody, -1, dtype=np.int32)
        for g in range(len(self.geom_bodyid) - 1, -1, -1):
            first[self.geom_bodyid[g]] = g
        return np.where(num > 0, first, -1).astype(np.int32)

    def key(self, name: str) -> np.ndarray:
        return self.key_qpos[self.names["key"].index(name)].copy()


def flatten(model) -> FlatModel:
    """Reduce an MjModel-like object (mink_b200.mjcf.Model or a real mujoco.MjModel) to a FlatModel."""
    nb, nj = int(model.nbody), int(model.njnt)
    parentid = np.asarray(model.body_parentid)
    jntadr, jntnum = np.asarray(model.body_jntadr), np.asarray(model.body_jntnum)
    bpos, bquat = np.asarray(model.body_pos, dtype=np.float64), np.asarray(model.body_quat, dtype=np.float64)
    jtype = np.asarray(model.jnt_type).astype(np.int32)

    ident_p, ident_q = np.zeros(3), np.array([1.0, 0.0, 0.0, 0.0])
    # Every body as (node, offset): node = last joint of the nearest jointed ancestor-or-self.
    body_frames: List[Frame] = [Frame(-1, ident_p.copy(), ident_q.copy())]
    node_parent = np.full(nj, -1, dtype=np.int32)
    node_pos = np.zeros((nj, 3))
    node_quat = np.tile(ident_q, (nj, 1))
    for b in range(1, nb):
        par = body_frames[parentid[b]]
        p, q = _compose(par.pos, par.quat, bpos[b], bquat[b] / np.linalg.norm(bquat[b]))
        if jntnum[b] == 0:
            body_frames.append(Frame(par.node, p, q))
            continue
        first = int(jntadr[b])
        node_parent[first] = par.node
        node_pos[first], node_quat[first] = p, q
        for j in range(first + 1, first + int(jntnum[b])):
            node_parent[j] = j - 1
        body_frames.append(Frame(first + int(jntnum[b]) - 1, ident_p.copy(), ident_q.copy()))

    qadr = np.asarray(model.jnt_qposadr).astype(np.int32)
    dadr = np.asarray(model.jnt_dofadr).astype(np.int32)
    nv, nq = int(model.nv), int(model.nq)
    dof_node = np.zeros(nv, dtype=np.int32)
    dof_qadr = np.full(nv, -1, dtype=np.int32)
    dof_limited = np.zeros(nv, dtype=np.int32)
    dof_lo = np.full(nv, -np.inf)
    dof_hi = np.full(nv, np.inf)
    limited = np.asarray(model.jnt_limited).astype(bool)
    rng = np.asarray(model.jnt_range, dtype=np.float64)
    for j in range(nj):
        t = int(jtype[j])
        for d in range(DOF_WIDTH[t]):
            dof_node[dadr[j] + d] = j
        if t in (JNT_SLIDE, JNT_HINGE):
            dof_qadr[dadr[j]] = qadr[j]
            if limited[j]:
                dof_limited[dadr[j]] = 1
                dof_lo[dadr[j]], dof_hi[dadr[j]] = rng[j]

    # CoM bookkeeping for mj_jacSubtreeCom(body=1) (reference com_task.py:69,82,96).
    com_node, com_pos, com_mass, com_missing = [], [], [], []
    missing = getattr(model, "body_mass_missing", None)   # only the MJCF-subset compiler sets it; a real MjModel has every mass
    names_body = getattr(model, "body_names", None)
    mass = np.asarray(model.body_mass, dtype=np.float64)
    ipos = np.asarray(model.body_ipos, dtype=np.float64)
    if nb > 1:
        for b in range(1, nb):
            a = b
            while a > 1:
                a = int(parentid[a])
            if a == 1 and missing is not None and missing[b]:
                com_missing.append(str(names_body[b]) if names_body is not None else str(b))
            if a != 1 or mass[b] <= 0.0:
                continue
            f = body_frames[b]
            com_node.append(f.node)
            com_pos.append(f.pos + _qrot(f.quat, ipos[b]))
            com_mass.append(mass[b])

    def attach(bodyids, lpos, lquat) -> List[Frame]:
        out = []
        for b, p, q in zip(bodyids, lpos, lquat):
            f = body_frames[int(b)]
            pp, qq = _compose(f.pos, f.quat, np.asarray(p, dtype=np.float64), np.asarray(q, dtype=np.float64))
            out.append(Frame(f.node, pp, qq))
        return out

    def names_of(kind, n):
        attr = {"body": "body_names", "joint": "joint_names", "geom": "geom_names",
                "site": "site_names", "key": "key_names"}[kind]
        if hasattr(model, attr):
            return list(getattr(model, attr))
        getter = getattr(model, kind)  # real mujoco.MjModel
        return [getter(i).name for i in range(n)]

    fm = FlatModel(
        nq=nq, nv=nv, nnode=nj,
        node_parent=node_parent, node_type=jtype, node_qadr=qadr, node_dadr=dadr,
        node_pos=node_pos, node_quat=node_quat,
        node_axis=np.asarray(model.jnt_axis, dtype=np.float64).reshape(nj, 3).copy(),
        node_jpos=np.asarray(model.jnt_pos, dtype=np.float64).reshape(nj, 3).copy(),
        qpos0=np.asarray(model.qpos0, dtype=np.float64).copy(),
        dof_node=dof_node, dof_qadr=dof_qadr, dof_limited=dof_limited, dof_lo=dof_lo, dof_hi=dof_hi,
        com_node=np.array(com_node, dtype=np.int32), com_pos=np.array(com_pos).reshape(-1, 3),
        com_mass=np.array(com_mass, dtype=np.float64),
    )
    fm.body_frames = body_frames
    fm.site_frames = attach(model.site_bodyid, model.site_pos, model.site_quat)
    fm.geom_frames = attach(model.geom_bodyid, model.geom_pos, model.geom_quat)
    fm.names = dict(body=names_of("body", nb), joint=names_of("joint", nj),
                    geom=names_of("geom", int(model.ngeom)), site=names_of("site", int(model.nsite)),
                    key=names_of("key", int(model.nkey)))
    fm.key_qpos = np.asarray(model.key_qpos, dtype=np.float64).reshape(-1, nq).copy()
    fm.com_missing = com_missing
    fm.geom_type = np.asarray(model.geom_type).astype(np.int32)
    fm.body_parentid = np.asarray(model.body_parentid).astype(np.int32)
    fm.geom_bodyid = np.asarray(model.geom_bodyid).astype(np.int32)
    fm.site_bodyid = np.asarray(model.site_bodyid).astype(np.int32)
    if getattr(model, "geom_contype", None) is not None:
        fm.geom_contype = np.asarray(model.geom_contype).astype(np.int32)
        fm.geom_conaffinity = np.asarray(model.geom_conaffinity).astype(np.int32)
    fm.geom_size = np.asarray(model.geom_size, dtype=np.float64).reshape(-1, 3).copy()
    fm.jnt_limited = limited.copy()
    fm.jnt_range = rng.copy()
    return fm


__all__ = ["FlatModel", "Frame", "flatten", "JNT_FREE", "JNT_BALL", "JNT_SLIDE", "JNT_HINGE",
           "QPOS_WIDTH", "DOF_WIDTH"]
