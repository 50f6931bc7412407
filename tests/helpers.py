"""Shared test helpers: load golden fixtures + flattened models (everything from tests/golden and mink_b200/models)."""

import os
import tarfile

import numpy as np

from mink_b200._abi import spec_from_workload
from mink_b200.workloads import WORKLOADS, load_flat, make_inputs, task_frames  # noqa: F401  (re-exported for the tests)

GOLDEN = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden")
# The MJCF files of the reference's example robots (meshes left out: the MJCF subset ignores them), each directory with the
# license it is distributed under.
EXAMPLE_SCENES = os.path.join(GOLDEN, "example_scenes.tar.xz")


def example_scene_files():
    """Paths of the example MJCF files, relative to the archive's root ("aloha/scene.xml", ...)."""
    with tarfile.open(EXAMPLE_SCENES) as tar:
        return sorted(n for n in tar.getnames() if n.endswith(".xml"))


def extract_example_scenes(dest: str) -> str:
    with tarfile.open(EXAMPLE_SCENES) as tar:
        tar.extractall(dest, filter="data")
    return dest


def load_case(name: str):
    wl = WORKLOADS[name]
    fm = load_flat(wl["robot"])
    spec = spec_from_workload(fm, wl)
    g = dict(np.load(os.path.join(GOLDEN, name + ".npz")))
    return wl, fm, spec, g


def track_case(name, B, T, seed, dtype, sigma=0.3):
    """A target sequence for the emulated converge / track loops: every hinge / slide moves from q0 by (t+1)/T of a random
    offset; the frame and CoM targets are the oracle's FK along that path.  Targets, q0 and the posture target in `dtype`."""
    from oracle.ikoracle import Oracle
    from tests.emu_lib import Emu

    wl, fm, spec, g = load_case(name)
    emu = Emu(fm.to_blob(), spec, fm.nq, fm.nv)
    orc = Oracle(fm.to_blob(), spec, fm.nq, fm.nv)
    frames = task_frames(wl, fm)
    fk = lambda qq: orc.fk(qq, frames)
    inp = make_inputs(fm, wl, B, fk, seed=seed, sigma=sigma)
    rng = np.random.default_rng(seed + 1)
    path = np.repeat(inp["q"][:, None, :], T, axis=1)
    frac = np.arange(1, T + 1) / T
    for n in range(fm.nnode):
        if int(fm.node_type[n]) >= 2:   # hinge / slide: q0 (+) (t+1)/T delta
            path[:, :, int(fm.node_qadr[n])] += rng.normal(0.0, sigma, size=B)[:, None] * frac[None, :]
    poses, com = fk(path.reshape(B * T, fm.nq))
    ft = np.asarray(poses, dtype).reshape(B, T, -1, 7)
    ct = np.asarray(com, dtype).reshape(B, T, -1, 3) if spec.ncom else None
    return dict(emu=emu, orc=orc, q0=inp["q"].astype(dtype), ft=ft, ct=ct, pt=inp["q"][:, None, :].astype(dtype),
                kw=dict(dt=wl["dt"], damping=wl["damping"]), B=B, T=T)


def chain_xml(n_hinge, *, free_base=False, ball=False, branch=0, collision=False, seed=0):
    """MJCF of a serial chain of `n_hinge` limited hinges (axes cycling x, y, z; short links with small random lateral
    offsets) ending in the site "tip".  free_base: a free joint at the root (6 leading dofs no limit bounds).  ball: one ball
    joint in the middle of the chain (nq = nv + 1).  branch: that many limited hinges in an untasked side branch hung off the
    middle of the chain (dofs the tip task does not couple, numbered between the chain's).  collision: a sphere on the tip
    and a capsule half-way up, next to a floor plane and a box."""
    rng = np.random.default_rng(seed)
    axes = ("1 0 0", "0 1 0", "0 0 1")

    def offset():
        dx, dy = rng.uniform(-0.015, 0.015, size=2)
        return f"{dx:.4f} {dy:.4f} 0.05"

    def hinge_body(name, k):
        return (f'<body name="{name}" pos="{offset()}"><joint name="{name}_j" type="hinge" axis="{axes[k % 3]}" range="-1.5 1.5" '
                f'limited="true"/><geom type="capsule" size="0.01 0.02" mass="0.1" contype="0" conaffinity="0"/>')

    mid = n_hinge // 2
    body, close = "", ""
    for i in range(n_hinge):
        body += hinge_body(f"b{i}", i)
        close += "</body>"
        if i == mid and branch:
            body += "".join(hinge_body(f"s{k}", k + 1) for k in range(branch)) + "</body>" * branch
        if i == mid and ball:
            body += f'<body name="ball" pos="{offset()}"><joint name="ball_j" type="ball"/><geom type="sphere" size="0.01" mass="0.1" contype="0" conaffinity="0"/>'
            close += "</body>"
        if i == mid and collision:
            body += '<geom name="mid" type="capsule" fromto="0 0 0 0 0 0.05" size="0.02"/>'
    tip = '<site name="tip" pos="0 0 0.05"/>'
    if collision:
        tip += '<geom name="tip_ball" type="sphere" size="0.03" pos="0 0 0.05"/>'
    root = body + tip + close
    if free_base:
        root = f'<body name="base" pos="0 0 0.4"><freejoint/><geom type="box" size="0.05 0.05 0.02" mass="1"/>{root}</body>'
    world = ('<geom name="floor" type="plane" size="5 5 0.1" pos="0 0 -0.3"/><geom name="wall" type="box" size="0.1 1 1" '
             'pos="0.6 0 0.5"/>' if collision else "")
    return f'<mujoco model="chain"><compiler angle="radian"/><worldbody>{world}{root}</worldbody></mujoco>'


def chain_case(n_hinge, *, free_base=False, ball=False, branch=0, collision=False, relative=False, seed=0):
    """A synthetic chain problem (chain_xml) as the driver sees it: a 6-D frame task on the tip, a posture task, a
    ConfigurationLimit and a VelocityLimit whose vmax differs from dof to dof (so that some bounds are active and some are
    not), plus the collision limit of the tip sphere and the mid capsule against the floor and the box when collision=True,
    and a RelativeFrameTask of the tip in the mid-chain body when relative=True (rows 6-11; its target is the second entry
    of the frame targets).  Returns a dict with the flat model, workload, spec, the tip frame, fk(q) through the fp64 oracle
    and, with relative=True, rel_frames = [tip, root] of the relative task."""
    import mink_b200 as mink
    from mink_b200._abi import LIMIT_VELOCITY
    from oracle.ikoracle import Oracle

    xml = chain_xml(n_hinge, free_base=free_base, ball=ball, branch=branch, collision=collision, seed=seed)
    fm = mink.flatten(mink.Model.from_xml_string(xml))
    limits = [dict(kind="configuration", gain=0.95), dict(kind="velocity", vmax=1.0)]
    if collision:
        limits.append(dict(kind="collision", pairs=[(["tip_ball", "mid"], ["floor", "wall"])], gain=0.85, minimum_distance=0.01,
                           detection_distance=0.3, bound_relaxation=0.0))
    wl = dict(robot="chain", key=None, frames=[dict(name="tip", type="site", position_cost=1.0, orientation_cost=1.0, lm_damping=1.0)],
              posture=dict(cost=1e-2), com=None, limits=limits, dt=2e-2, damping=1e-3)
    if relative:
        wl["relative_frames"] = [dict(name="tip", type="site", root_name=f"b{n_hinge // 2}", root_type="body", position_cost=1.0,
                                      orientation_cost=1.0, lm_damping=1.0)]
    spec = spec_from_workload(fm, wl)
    rng = np.random.default_rng(seed + 1000)
    for lim in spec.limits:
        if lim.kind == LIMIT_VELOCITY:   # 0.75 .. 12 rad/s, i.e. a bound of 0.015 .. 0.24 rad per step
            lim.vmax = np.exp(rng.uniform(np.log(0.75), np.log(12.0), size=len(lim.dof)))
    frames = task_frames(wl, fm)
    orc = Oracle(fm.to_blob(), spec, fm.nq, fm.nv)
    out = dict(xml=xml, fm=fm, wl=wl, spec=spec, frames=frames, orc=orc, fk=lambda qq: orc.fk(qq, frames))
    if relative:
        out["rel_frames"] = [fm.frame(f[k + "name"], f[k + "type"]) for f in wl["relative_frames"] for k in ("", "root_")]
    return out


# The chain_case problems on both sides of every switch of K2's dispatch: id -> (chain_case keyword arguments, coupled dofs
# nu, unbounded leading dofs nfree).  nu = 8 / 9: G = 4 -> 8 lanes per problem; 32 / 33: 32-bit -> 64-bit active-set masks;
# 64: the widest block; nu + 1 = 8, 16, 32, 64, 65: the general path's lanes per problem and slots per lane.  With collision
# rows every dof is coupled and the general path solves.
CHAIN_CASES = {f"n{n}": (dict(n_hinge=n), n, 0) for n in (1, 7, 8, 9, 15, 16, 31, 32, 33, 63, 64)}
CHAIN_CASES.update({
    "free32": (dict(n_hinge=26, free_base=True), 32, 6),
    "free64": (dict(n_hinge=58, free_base=True), 64, 6),
    "ball64": (dict(n_hinge=61, ball=True), 64, 0),          # nq = 65
    "branch33": (dict(n_hinge=33, branch=31), 33, 0),        # nv = 64, the side branch is not coupled
})
CHAIN_CASES.update({f"coll{n}": (dict(n_hinge=n, collision=True), n, 0) for n in (31, 32, 63, 64)})


def chain_case_by_id(cid):
    kw, nu, nfree = CHAIN_CASES[cid]
    return chain_case(seed=nu, **kw)


def assert_chain_uses_top_of_block(c, nu, q, step_out):
    """On the oracle's optimum (Oracle.step's output for q): the last coupled dof (the tip hinge, numbered last in every
    chain layout) is at a bound in some instances and free in others, and the mean active count lies strictly between 0 and
    nu -- so the top bit of the active-set masks and the top slot of the factor carry real work."""
    dq, _, st, nact = step_out
    assert not st.any()
    lo, hi = c["orc"].box(q, c["wl"]["dt"])
    last = c["fm"].nv - 1
    at_bound = (np.abs(dq[:, last] - lo[:, last]) < 1e-9) | (np.abs(dq[:, last] - hi[:, last]) < 1e-9)
    assert at_bound.any() and not at_bound.all(), at_bound.mean()
    assert 0 < nact.mean() < nu, nact.mean()


def qmul_np(a, b):
    """Hamilton product of (..., 4) quaternion arrays (w, x, y, z)."""
    w1, x1, y1, z1 = np.moveaxis(np.asarray(a), -1, 0)
    w2, x2, y2, z2 = np.moveaxis(np.asarray(b), -1, 0)
    return np.stack([w1 * w2 - x1 * x2 - y1 * y2 - z1 * z2, w1 * x2 + x1 * w2 + y1 * z2 - z1 * y2,
                     w1 * y2 - x1 * z2 + y1 * w2 + z1 * x2, w1 * z2 + x1 * y2 - y1 * x2 + z1 * w2], -1)


def qrot_np(q, v):
    """Rotate (..., 3) vectors by unit (..., 4) quaternions."""
    u = np.asarray(q)[..., 1:]
    t = 2 * np.cross(u, v)
    return v + np.asarray(q)[..., :1] * t + np.cross(u, t)


def targets_at_angle(pose, theta, offset, rng):
    """Targets T_t = T (R, d) for poses T [B, 7] (w, x, y, z, px, py, pz): a rotation R of exactly `theta` rad about a
    random unit axis per instance, then a body-frame translation d of length `offset` in a random direction.  The error
    log(T^-1 T_t) of a FrameTask at T then has angle `theta`.  At theta == pi the rotation's w
    is exactly 0, so either sign of the log is valid."""
    pose = np.asarray(pose, np.float64)
    B = pose.shape[0]
    ax = rng.normal(size=(B, 3))
    ax /= np.linalg.norm(ax, axis=1, keepdims=True)
    d = rng.normal(size=(B, 3))
    d *= offset / np.linalg.norm(d, axis=1, keepdims=True)
    c, s = (0.0, 1.0) if theta == np.pi else (np.cos(theta / 2), np.sin(theta / 2))
    rot = np.concatenate([np.full((B, 1), c), s * ax], 1)
    return np.concatenate([qmul_np(pose[:, :4], rot), pose[:, 4:] + qrot_np(pose[:, :4], d)], 1)


def quat_align(a, b):
    """Flip sign of quaternions in a (...,4) to match b's hemisphere."""
    s = np.sign(np.sum(a * b, axis=-1, keepdims=True))
    s[s == 0] = 1
    return a * s


# The Lie layer's regimes (mink_b200/csrc/bik_math.h): 0 and 1e-9 (identity branch of the Jacobian, |w|^2 < 1e-10), 1e-5 (1 -/+ 1e-3)
# on both sides of that switch, the Maclaurin series up to theta^2 = 1 with 1 -/+ 1e-6 on both sides of its switch, the closed
# forms above it, and the log's branch flip at pi.  Offsets: the target's translation from the frame, in m.
LIE_ANGLES = (0.0, 1e-9, 1e-5 * (1 - 1e-3), 1e-5 * (1 + 1e-3), 1e-4, 1e-3, 0.3, 0.7, 1 - 1e-6, 1 + 1e-6, 1.5, 2.5, 3.0,
              np.pi - 1e-2, np.pi - 1e-3)
LIE_OFFSETS = (0.0, 1e-6, 0.3)
# chain_case keyword arguments: a hinge chain, a free base with 26 hinges, a ball joint in a 61-hinge chain, and the tip
# relative to a mid-chain body besides the absolute tip task
LIE_CASES = {"n7": dict(n_hinge=7), "free32": dict(n_hinge=26, free_base=True), "ball64": dict(n_hinge=61, ball=True),
             "rel7": dict(n_hinge=7, relative=True)}


def lie_case(cid):
    return chain_case(seed=7, **LIE_CASES[cid])


def lie_targets(c, q, theta, offset, rng):
    """Frame targets [B, F, 7] at `theta` rad and `offset` m from every frame task's current pose at q (targets_at_angle),
    the relative task's in its root frame."""
    poses, _ = c["orc"].fk(q, c["frames"], want_com=False)
    ft = [targets_at_angle(poses[:, 0], theta, offset, rng)]
    if "rel_frames" in c:
        pr, _ = c["orc"].fk(q, c["rel_frames"], want_com=False)
        qrc = pr[:, 1, :4] * np.array([1.0, -1.0, -1.0, -1.0])
        rel = np.concatenate([qmul_np(qrc, pr[:, 0, :4]), qrot_np(qrc, pr[:, 0, 4:] - pr[:, 1, 4:])], 1)
        ft.append(targets_at_angle(rel, theta, offset, rng))
    return np.stack(ft, 1)


def lie_task_rows(c, q, ft, e_like=None):
    """(e [B, 6F], J [B, 6F, nv]) of the frame tasks at q, ft from tests/lie_ref: the oracle's fp64 FK and body Jacobians,
    the Lie layer in extended precision.  e_like [B, 6F], a kernel's e: see tests/lie_ref.frame_task."""
    from tests import lie_ref

    orc = c["orc"]
    poses, _ = orc.fk(q, c["frames"], want_com=False)
    Jb = orc.frame_jacobian(q, c["frames"])
    sl = lambda k: None if e_like is None else e_like[:, 6 * k:6 * k + 6]
    e, J = lie_ref.frame_task(poses[:, 0], Jb[:, 0], ft[:, 0], sl(0))
    es, Js = [e], [J]
    if "rel_frames" in c:
        pr, _ = orc.fk(q, c["rel_frames"], want_com=False)
        Jr = orc.frame_jacobian(q, c["rel_frames"])
        e, J = lie_ref.relative_frame_task(pr[:, 0], Jr[:, 0], pr[:, 1], Jr[:, 1], ft[:, 1], sl(1))
        es.append(e); Js.append(J)
    return np.concatenate(es, 1), np.concatenate(Js, 1)
