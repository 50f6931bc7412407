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


def quat_align(a, b):
    """Flip sign of quaternions in a (...,4) to match b's hemisphere."""
    s = np.sign(np.sum(a * b, axis=-1, keepdims=True))
    s[s == 0] = 1
    return a * s
