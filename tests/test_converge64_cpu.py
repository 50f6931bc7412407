"""bik_converge64 / bik_track64's pass loops with the kernel headers compiled for the host (tests/host_emu), no GPU needed.

The fp64 loops run the fp64 K1 and K2's fp64-I/O forms on fp64 buffers, collision rows included, so they are held to the
oracle's own bars rather than to fp32 ones: the golden converge loops with identical iteration counts and flags, track64
bit-equal to the per-frame converge64 loop, and every iteration count of a ragged batch equal to the C oracle's.
"""

import numpy as np
import pytest

from tests.emu_lib import Emu
from tests.helpers import load_case, track_case

CASES = ["ur5e", "ur5e_dls", "g1", "shadow", "spot", "g1_rel", "edge", "g1_full", "g1_hands", "ur5e_damp", "ur5e_wall",
         "iiwa", "h1", "go1", "stretch", "tidybot", "aloha", "aloha_coll", "leap"]
# the oracle's bars in tests/test_oracle_golden.py::test_converge_loop, times 10
GOLDEN_TOL = {"spot": 1e-3, "g1_rel": 1e-4, "edge": 1e-5}
CONV = dict(max_iters=10, pos_threshold=2e-3, ori_threshold=2e-3)


@pytest.mark.parametrize("name", CASES)
def test_emulated_converge64_matches_golden_loops(name):
    wl, fm, spec, g = load_case(name)
    emu = Emu(fm.to_blob(), spec, fm.nq, fm.nv)
    CB = g["conv_q"].shape[0]
    max_iters, pos, ori = int(g["conv_params"][0]), float(g["conv_params"][1]), float(g["conv_params"][2])
    ct = g["com_target"][:CB] if "com_target" in g else None
    q, it, st = emu.converge(g["q"][:CB], g["frame_targets"][:CB], g["posture_target"], ct, dt=float(g["dt"]),
                             damping=float(g["damping"]), max_iters=max_iters, pos_threshold=pos, ori_threshold=ori)
    assert q.dtype == np.float64
    assert int((st & 15).max()) == 0
    np.testing.assert_array_equal(it, g["conv_iters"])
    np.testing.assert_array_equal((st & 16) == 0, g["conv_ok"].astype(bool))
    err = np.abs(q - g["conv_q"]).max()
    print(f"{name}: max|q - q_golden| = {err:.2e} (bar {GOLDEN_TOL.get(name, 1e-6):.0e})")
    assert err <= GOLDEN_TOL.get(name, 1e-6)


@pytest.mark.parametrize("name", ["ur5e", "h1", "ur5e_wall", "spot"])
def test_emulated_track64_equals_per_frame_converge64(name):
    """ur5e: small-group K2; h1: CoM trajectory; ur5e_wall: collision rows, general K2; spot: the ill-conditioned case."""
    c = track_case(name, B=64 + 5, T=6, seed=12, dtype=np.float64)
    B, T = c["B"], c["T"]
    ln = np.random.default_rng(2).integers(0, T + 1, size=B).astype(np.int32)
    ln[:3] = [0, T, 1]
    q = c["q0"]
    q_loop, it_loop, st_loop = np.zeros((B, T, q.shape[1])), np.zeros((B, T), np.int32), np.zeros((B, T), np.int32)
    for t in range(T):
        q, it_loop[:, t], st_loop[:, t] = c["emu"].converge(q, c["ft"][:, t], c["pt"], None if c["ct"] is None else c["ct"][:, t],
                                                            **c["kw"], **CONV)
        q_loop[:, t] = q
    q_end, q_traj, it, st, passes = c["emu"].track(c["q0"], c["ft"], c["pt"], c["ct"], **c["kw"], **CONV, lengths=ln)
    assert q_traj.dtype == np.float64
    has = np.arange(T)[None, :] < ln[:, None]
    np.testing.assert_array_equal(q_traj[has], q_loop[has])
    np.testing.assert_array_equal(it[has], it_loop[has])
    np.testing.assert_array_equal(st[has], st_loop[has])
    assert np.isnan(q_traj[~has]).all() and (it[~has] == -1).all() and (st[~has] == -1).all()
    q_ref = np.where(ln[:, None] > 0, q_loop[np.arange(B), np.maximum(ln - 1, 0)], c["q0"])
    np.testing.assert_array_equal(q_end, q_ref)
    assert passes == int(np.where(has, it + 1, 0).sum(1).max())
    print(f"{name}: iters histogram {np.bincount(it[has]).tolist()} passes {passes}")


def test_emulated_track64_against_oracle():
    """The oracle's fp64 converge loop, frame after frame, on a ragged UR5e batch: every iteration count is the same and
    q_traj is within 1e-6."""
    c = track_case("ur5e", B=200 + 3, T=8, seed=44, dtype=np.float64)
    B, T = c["B"], c["T"]
    ln = np.random.default_rng(4).integers(0, T + 1, size=B).astype(np.int32)
    ln[:3] = [0, T, 1]
    _, q_traj, it, st, _ = c["emu"].track(c["q0"], c["ft"], c["pt"], None, **c["kw"], **CONV, lengths=ln)
    q = c["q0"].copy()
    q_ref, it_ref, ok_ref = np.zeros(q_traj.shape), np.zeros_like(it), np.zeros(it.shape, bool)
    for t in range(T):
        q, it_ref[:, t], ok_ref[:, t], _ = c["orc"].converge(q, c["ft"][:, t], c["pt"], None, **c["kw"], **CONV)
        q_ref[:, t] = q
    has = np.arange(T)[None, :] < ln[:, None]
    # the oracle runs every frame for every instance; an instance's frames up to its length are the same computation
    print(f"track64 vs oracle: {int((it[has] != it_ref[has]).sum())} of {int(has.sum())} iteration counts differ, "
          f"max|q - q_oracle| {np.abs(q_traj[has] - q_ref[has]).max():.2e}")
    np.testing.assert_array_equal(it[has], it_ref[has])
    np.testing.assert_array_equal(((st & 16) == 0)[has], ok_ref[has])
    np.testing.assert_allclose(q_traj[has], q_ref[has], atol=1e-6)
