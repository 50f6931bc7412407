"""Kernel math (mink_b200/csrc headers compiled for the host, one lane) vs the golden vectors.

fp32 device arithmetic against the fp64 reference: tolerances are the fp64->fp32 budget stated in
BASELINE.json (dq within 1e-4 rad) and tighter where the quantity allows it.  The GPU tests repeat
these checks through the real kernels; this file lets the math be debugged without a GPU.
"""

import numpy as np
import pytest

from tests.emu_lib import Emu
from mink_b200.workloads import make_inputs
from tests.helpers import load_case, quat_align, task_frames

CASES = ["ur5e", "ur5e_dls", "g1", "shadow", "spot", "g1_rel", "edge", "g1_full", "g1_hands", "ur5e_damp", "ur5e_wall",
         "iiwa", "h1", "go1", "stretch", "tidybot", "aloha", "aloha_coll", "leap"]   # the last eight: the reference's other example robots


def _emu(name):
    wl, fm, spec, g = load_case(name)
    return wl, fm, spec, g, Emu(fm.to_blob(), spec, fm.nq, fm.nv)


@pytest.mark.parametrize("name", CASES)
def test_fk_and_body_jacobian(name):
    wl, fm, spec, g, emu = _emu(name)
    frames = task_frames(wl, fm)
    poses, com, Jb = emu.fk(g["q"], frames, want_J=True)
    ref = g["frame_pose"][:, :len(frames)]
    np.testing.assert_allclose(poses[..., 4:], ref[..., 4:], atol=5e-6)
    np.testing.assert_allclose(quat_align(poses[..., :4].astype(np.float64), ref[..., :4]), ref[..., :4], atol=5e-6)
    np.testing.assert_allclose(Jb, g["J_body"][:, :len(frames)], atol=1e-5)
    if fm.ncom:
        np.testing.assert_allclose(com, g["com"], atol=5e-6)


@pytest.mark.parametrize("name", CASES)
def test_k1_errors_and_jacobians(name):
    wl, fm, spec, g, emu = _emu(name)
    J, e, ep, Gc, hc = emu.fk_jac(g["q"], g["frame_targets"], g["posture_target"], g.get("com_target"), dt=float(g["dt"]))
    F = spec.nframe
    np.testing.assert_allclose(e[:, :6 * F].reshape(-1, F, 6), g["e_frame"], atol=2e-5)
    np.testing.assert_allclose(J[:, :6 * F].reshape(-1, F, 6, fm.nv), g["J_frame"], atol=5e-5)
    if spec.nposture:
        np.testing.assert_allclose(ep[:, 0], g["e_posture"], atol=1e-6)
    if spec.ncom:
        np.testing.assert_allclose(e[:, 6 * F:], g["e_com"], atol=5e-6)
        np.testing.assert_allclose(J[:, 6 * F:], g["J_com"], atol=5e-6)
    if spec.npairs:
        Gr, hr = g["G"][:, -spec.npairs:], g["h"][:, -spec.npairs:]   # collision rows are stacked last
        fin = np.isfinite(hr)
        assert np.array_equal(np.isfinite(hc), fin)
        np.testing.assert_allclose(hc[fin], hr[fin], rtol=2e-4, atol=2e-3)
        # capsule-capsule closest POINTS are ill-conditioned when the axes are nearly parallel (the distance is
        # not): fp32 poses move the contact point along the segment, hence the looser bound for that model
        np.testing.assert_allclose(Gc, Gr, atol=2e-5 if name != "edge" else 5e-3)


@pytest.mark.parametrize("name", CASES)
def test_k2_from_golden_jacobians(name):
    """K2 alone: feed the reference's own (J, e) cast to fp32, compare H, c, box and dq."""
    wl, fm, spec, g, emu = _emu(name)
    B, F = g["q"].shape[0], spec.nframe
    J = np.concatenate([g["J_frame"].reshape(B, 6 * F, fm.nv)] + ([g["J_com"]] if spec.ncom else []), axis=1)
    e = np.concatenate([g["e_frame"].reshape(B, 6 * F)] + ([g["e_com"]] if spec.ncom else []), axis=1)
    ep = g["e_posture"][:, None, :] if spec.nposture else np.zeros((B, 0, fm.nv))
    if spec.npairs:
        Gc, hc = g["G"][:, -spec.npairs:], g["h"][:, -spec.npairs:]
    else:
        Gc, hc = np.zeros((B, 0, fm.nv)), np.zeros((B, 0))
    dq, st, it, H, c, lo, hi = emu.solve(g["q"], J, e, ep, Gc, hc, float(g["dt"]), float(g["damping"]),
                                         use_double=True, want_objective=True)
    assert not st.any(), st
    scale = np.abs(g["H"]).max()
    np.testing.assert_allclose(H, g["H"], atol=1e-6 * scale)
    np.testing.assert_allclose(c, g["c"], atol=1e-5 * max(1.0, np.abs(g["c"]).max()))
    fin = np.isfinite(g["box_lo"])
    np.testing.assert_allclose(lo[fin], g["box_lo"][fin], atol=1e-6)
    fin = np.isfinite(g["box_hi"])
    np.testing.assert_allclose(hi[fin], g["box_hi"][fin], atol=1e-6)
    tol = 2e-3 if name == "spot" else 1e-5   # Spot: cond(H) ~ 4e7, fp32 inputs alone move the optimum
    np.testing.assert_allclose(dq, g["dq"], atol=tol)


@pytest.mark.parametrize("name", CASES)
def test_full_step(name):
    """K1 -> K2 -> integrate in fp32 I/O against the reference's solve_ik + integrate."""
    wl, fm, spec, g, emu = _emu(name)
    dt, damping = float(g["dt"]), float(g["damping"])
    J, e, ep, Gc, hc = emu.fk_jac(g["q"], g["frame_targets"], g["posture_target"], g.get("com_target"), dt=dt)
    dq, st, it, *_ = emu.solve(g["q"], J, e, ep, Gc, hc, dt, damping, use_double=True)
    assert not st.any()
    tol = {"spot": 5e-3, "g1_rel": 1e-4 * max(1.0, np.abs(g["dq"]).max()),
           "edge": 2e-3}.get(name, 1e-4)   # edge: an active near-parallel capsule pair (ill-conditioned contact point)
    err = np.abs(dq - g["dq"]).max()
    print(name, "max |dq - dq_ref| =", err, "iters mean/max", it.mean(), it.max())
    assert err < tol
    qn = emu.integrate(g["q"], dq)
    np.testing.assert_allclose(qn, g["q_next"], atol=2 * tol)


@pytest.mark.parametrize("name", ["g1", "ur5e", "ur5e_dls", "shadow", "g1_rel"])
@pytest.mark.parametrize("code", [3, 8])
def test_small_paths_match_reference(name, code):
    """K2 small-group path (3: 32-bit masks, 8: the 64-bit masks of the wide instantiation): same optimum as the warp path
    and the reference."""
    wl, fm, spec, g, emu = _emu(name)
    dt, damping = float(g["dt"]), float(g["damping"])
    J, e, ep, Gc, hc = emu.fk_jac(g["q"], g["frame_targets"], g["posture_target"], None, dt=dt)
    dq, st, it, *_ = emu.solve(g["q"], J, e, ep, Gc, hc, dt, damping, use_double=code)
    assert not st.any()
    err = np.abs(dq - g["dq"]).max()
    print(name, "thread path max |dq - dq_ref| =", err, "iters mean/max", it.mean(), it.max())
    tol = 1e-4 * max(1.0, np.abs(g["dq"]).max())
    assert err < tol
    dq_dense, _, it_dense, *_ = emu.solve(g["q"], J, e, ep, Gc, hc, dt, damping, use_double=1)
    np.testing.assert_allclose(dq, dq_dense, atol=2e-6)
    if code == 3:   # Gauss-Seidel guess + primal active set: same optimum; the iteration count is informational
        print(name, "pivoting iterations small-group", it.sum(), "dense cold start", it_dense.sum())


def test_check_limits():
    wl, fm, spec, g, emu = _emu("g1")
    q = g["q"].copy()
    assert not emu.check_limits(q).any()
    q[3, 10] = 100.0
    st = emu.check_limits(q)
    assert st[3] == 1 and st.sum() == 1


def test_image_marks_unbounded_leading_dofs_and_compact_state():
    """K2 eliminates the leading coupled dofs that no limit bounds once (the free joint of G1: mink/limits/
    configuration_limit.py:40-56 and velocity_limit.py:47-60 skip free joints); K1's pose state has one row per
    VISITED node unless a CoM task / collision limit indexes by node id."""
    h = _emu("g1")[4].header()
    assert (h["nu"], h["nfree"]) == (18, 6)            # floating base + two legs coupled; the base has no bounds
    assert h["nslots"] == h["nneeded"] == 13 and h["nnode"] == 38
    h = _emu("ur5e_dls")[4].header()
    assert h["nfree"] == h["nu"] == 6                  # limits=[]: the elimination is the whole solve
    h = _emu("ur5e")[4].header()
    assert h["nfree"] == 0 and h["nu"] == 6
    h = _emu("shadow")[4].header()
    assert h["nfree"] == 0
    h = _emu("spot")[4].header()
    assert h["nfree"] == 0 and h["nslots"] == h["nnode"]   # collision rows + CoM task: general path, identity slots


def test_unbounded_elimination_matches_full_pivoting_with_active_bounds():
    """The G1 golden has active velocity bounds: the reduced (Schur complement) pivoting, started from the projected
    Gauss-Seidel guess, must land on the reference's optimum in fewer pivoting iterations than the dense path needs on
    the whole coupled block from a cold start."""
    wl, fm, spec, g, emu = _emu("g1")
    dt, damping = float(g["dt"]), float(g["damping"])
    J, e, ep, Gc, hc = emu.fk_jac(g["q"], g["frame_targets"], g["posture_target"], None, dt=dt)
    dq, st, it, *_ = emu.solve(g["q"], J, e, ep, Gc, hc, dt, damping, use_double=3)
    dq_dense, _, it_dense, *_ = emu.solve(g["q"], J, e, ep, Gc, hc, dt, damping, use_double=1)
    assert not st.any() and it_dense.max() > 1
    assert it.mean() < 0.5 * it_dense.mean()
    np.testing.assert_allclose(dq, dq_dense, atol=1e-7)
    np.testing.assert_allclose(dq, g["dq"], atol=1e-5)


def test_small_group_path_at_its_size_limit():
    """g1_hands (the reference's humanoid example without the CoM task): 31 coupled dofs -- the largest block whose active
    set fits the 32-bit masks of the small-group path -- 6 of them unbounded, 18 bounds active on average."""
    wl, fm, spec, g, emu = _emu("g1_hands")
    h = emu.header()
    assert (h["nu"], h["nfree"]) == (31, 6)
    dt, damping = float(g["dt"]), float(g["damping"])
    J, e, ep, Gc, hc = emu.fk_jac(g["q"], g["frame_targets"], g["posture_target"], None, dt=dt)
    ref, _, it_dense, *_ = emu.solve(g["q"], J, e, ep, Gc, hc, dt, damping, use_double=1)
    for sweeps in (3, 8):
        emu.set_knobs(sweeps)
        dq, st, it, *_ = emu.solve(g["q"], J, e, ep, Gc, hc, dt, damping, use_double=3)
        assert not st.any()
        np.testing.assert_allclose(dq, ref, atol=2e-6)
        assert np.abs(dq - g["dq"]).max() < 1e-4 * max(1.0, np.abs(g["dq"]).max())
        print("g1_hands sweeps", sweeps, "iters mean/max", it.mean(), it.max(), "(dense cold:", it_dense.mean(), it_dense.max(), ")")


def test_rollout_with_carried_state_converges_and_matches_oracle():
    """The regime the reference's examples run in (examples/humanoid_g1.py:81-94: solve_ik + integrate, targets held).
    From the second step on block principal pivoting stalls on a few instances per thousand (the single-pivot fallback
    runs out of iterations); the small-group path therefore starts a primal active-set method from the previous step's dq
    (clipped, polished by Gauss-Seidel sweeps).  Every instance must converge at every step and match the exact
    Goldfarb-Idnani oracle (the algorithm quadprog implements)."""
    from oracle.ikoracle import Oracle

    wl, fm, spec, g, emu = _emu("g1")
    frames = task_frames(wl, fm)
    orc = Oracle(fm.to_blob(), spec, fm.nq, fm.nv)
    B, T = 768, 8

    def fk(qq):
        p, c, _ = emu.fk(qq, frames)
        return p.astype(np.float64), c.astype(np.float64)

    inp = make_inputs(fm, wl, B, fk, seed=77)
    q = inp["q"].astype(np.float32)
    warm = np.zeros((B, emu.header()["nu"]), np.int8)
    dq = np.full((B, fm.nv), np.nan, np.float32)    # whatever the caller's buffer held before the first step
    worst = 0
    for step in range(T):
        J, e, ep, Gc, hc = emu.fk_jac(q, inp["frame_targets"], inp["posture_target"], None, dt=wl["dt"])
        dq, st, it = emu.solve_warm(q, J, e, ep, wl["dt"], wl["damping"], dq, warm)
        dq_ref, _, st_ref, _ = orc.step(q.astype(np.float64), inp["frame_targets"], inp["posture_target"], None, dt=wl["dt"],
                                        damping=wl["damping"], nsteps=1, integrate=False)
        assert not st.any() and not st_ref.any(), (step, np.flatnonzero(st))
        assert np.abs(dq - dq_ref).max() < 1e-4
        assert (warm[:, 0] & 4).all()
        worst = max(worst, int(it.max()))
        q = emu.integrate(q, dq)
    print("rollout: worst pivoting iteration count", worst)
    assert worst <= 30


def _k2_path(emu):
    h = emu.header()
    if emu.spec.npairs:
        return 1
    return 8 if h["nu"] > 32 else 3


@pytest.mark.parametrize("name", CASES)
def test_packed_handoff_matches_dense(name):
    """bik_step's K1 -> K2 hand-off (non-zero columns only, posture error recomputed by K2) gives the dq of the dense
    Task.compute_jacobian form; the fused check_limits reports the same bits as the stand-alone one."""
    wl, fm, spec, g, emu = _emu(name)
    dt, damping = float(g["dt"]), float(g["damping"])
    args = (g["q"], g["frame_targets"], g["posture_target"], g.get("com_target"))
    J, e, ep, Gc, hc = emu.fk_jac(*args, dt=dt)
    pk, Gc2, hc2, st1 = emu.fk_jac(*args, dt=dt, packed=True, check=True)
    assert not np.isnan(pk[:, :emu.header()["pk_stride"] - 3]).any()   # every entry of the record is written (tail = alignment padding)
    np.testing.assert_array_equal(Gc, Gc2)
    np.testing.assert_array_equal(st1, emu.check_limits(g["q"]))
    path = _k2_path(emu)
    dq_d, st_d, *_ = emu.solve(g["q"], J, e, ep, Gc, hc, dt, damping, use_double=path)
    dq_p, st_p, it, H, c, lo, hi, q_next = emu.solve(g["q"], None, None, None, Gc, hc, dt, damping, use_double=path, pk=pk,
                                                     ptgt=g["posture_target"], integrate=True)
    assert not st_d.any() and not st_p.any()
    np.testing.assert_allclose(dq_p, dq_d, atol=1e-7)
    np.testing.assert_allclose(q_next, emu.integrate(g["q"], dq_p), atol=1e-6)


@pytest.mark.parametrize("name", CASES)
def test_fp64_path_reproduces_the_reference(name):
    """fp64 instantiation of K1 (fp64 kinematic constants, fp64 inputs) + fp64 hand-off + fp64 K2 + fp64 dq: the
    reference's numbers to solver tolerance, ill-conditioned configurations (Spot: cost 200 against damping 1e-3)
    included -- the reference is fp64 end to end (mink/solve_ik.py:13-22)."""
    wl, fm, spec, g, emu = _emu(name)
    dt, damping = float(g["dt"]), float(g["damping"])
    args = (g["q"], g["frame_targets"], g["posture_target"], g.get("com_target"))
    J, e, ep, Gc, hc = emu.fk_jac(*args, dt=dt, prec="f64")
    F = spec.nframe
    np.testing.assert_allclose(e[:, :6 * F].reshape(-1, F, 6), g["e_frame"], atol=1e-10)
    np.testing.assert_allclose(J[:, :6 * F].reshape(-1, F, 6, fm.nv), g["J_frame"], atol=1e-9)
    if spec.nposture:
        np.testing.assert_allclose(ep[:, 0], g["e_posture"], atol=1e-12)
    if spec.ncom:
        np.testing.assert_allclose(e[:, 6 * F:], g["e_com"], atol=1e-12)
        np.testing.assert_allclose(J[:, 6 * F:], g["J_com"], atol=1e-12)
    if spec.npairs:
        Gr, hr = g["G"][:, -spec.npairs:], g["h"][:, -spec.npairs:]
        fin = np.isfinite(hr)
        assert np.array_equal(np.isfinite(hc), fin)
        np.testing.assert_allclose(hc[fin], hr[fin], rtol=1e-9, atol=1e-9)
        np.testing.assert_allclose(Gc, Gr, atol=1e-9)
    pk, Gc, hc = emu.fk_jac(*args, dt=dt, prec="f64", packed=True)
    dq, st, it, H, c, lo, hi, q_next = emu.solve(g["q"], None, None, None, Gc, hc, dt, damping, use_double=_k2_path(emu), io64=True,
                                                 pk=pk, ptgt=g["posture_target"], integrate=True)
    assert not st.any()
    err = np.abs(dq - g["dq"]).max()
    print(name, "fp64 path max |dq - dq_ref| =", err, "iters mean/max", it.mean(), it.max())
    assert err < 2e-7 * max(1.0, np.abs(g["dq"]).max())   # bounds are kept in fp32 (1e-7 relative)
    np.testing.assert_allclose(q_next, g["q_next"], atol=1e-6)


@pytest.mark.parametrize("name", ["spot", "edge", "shadow"])
def test_fp64_kernel_on_fp32_inputs_matches_oracle_on_the_same_inputs(name):
    """What bik_step runs for an ill-conditioned problem of an fp32 caller: inputs rounded to fp32, everything downstream
    in fp64.  Checked against the oracle evaluated ON THE ROUNDED INPUTS (identical inputs, north_star): the rounding of q
    itself moves Spot's optimum by ~1e-4 (cost / (2 sqrt(damping)) ~ 3e3 times 3e-8), which no kernel can undo."""
    from oracle.ikoracle import Oracle

    wl, fm, spec, g, emu = _emu(name)
    dt, damping = float(g["dt"]), float(g["damping"])
    r32 = lambda a: None if a is None else np.asarray(a, np.float32).astype(np.float64)
    q, ft, pt, ct = r32(g["q"]), r32(g["frame_targets"]), r32(g["posture_target"]), r32(g.get("com_target"))
    orc = Oracle(fm.to_blob(), spec, fm.nq, fm.nv)
    dq_ref, _, st_ref, _ = orc.step(q, ft, pt, ct, dt=dt, damping=damping, nsteps=1, integrate=False)
    pk, Gc, hc = emu.fk_jac(q, ft, pt, ct, dt=dt, prec="mixed", packed=True)
    dq, st, it, *_ = emu.solve(q, None, None, None, Gc, hc, dt, damping, use_double=_k2_path(emu), pk=pk, ptgt=pt)
    assert not st.any() and not st_ref.any()
    err = np.abs(dq - dq_ref).max()
    print(name, "fp64 kernels on fp32 inputs: max |dq - dq_oracle(same inputs)| =", err)
    assert err < 1e-5


def test_inconsistent_limits_are_flagged():
    """A limited dof 1 rad past its upper limit with a velocity limit: ConfigurationLimit wants dq <= -0.95, VelocityLimit
    dq >= -dt*vmax -- the reference hands qpsolvers an infeasible QP (solve_ik.py:103 asserts).  Every K2 path must set
    BIK_STATUS_QP_INFEASIBLE instead of returning a dq that breaks the velocity limit."""
    wl, fm, spec, g, emu = _emu("g1")
    dt, damping = float(g["dt"]), float(g["damping"])
    q = g["q"][:4].copy()
    d = 20
    qa = int(fm.dof_qadr[d])
    q[1, qa] = fm.dof_hi[d] + 1.0
    args = (q, g["frame_targets"][:4], g["posture_target"], None)
    J, e, ep, Gc, hc = emu.fk_jac(*args, dt=dt)
    for path in (1, 3, 8):
        dq, st, *_ = emu.solve(q, J, e, ep, Gc, hc, dt, damping, use_double=path)
        assert st[1] & 8 and not (st[[0, 2, 3]] & 8).any(), (path, st)


def test_more_active_collision_rows_than_the_solver_holds_are_flagged():
    """K2 keeps at most K2_MAX_GEN (24) general rows active at once.  A problem that needs more -- here Spot's four foot/floor
    pairs listed ten times over, all pushed into the floor -- must come back flagged (BIK_STATUS_QP_MAXITER), never as a
    silently truncated "solution" (round-1 advisor finding)."""
    from mink_b200._abi import spec_from_workload
    from mink_b200.workloads import WORKLOADS

    wl = dict(WORKLOADS["spot"])
    wl["limits"] = [dict(WORKLOADS["spot"]["limits"][0], pairs=[(["FL", "FR", "HR", "HL"], ["floor"])] * 10)]
    _, fm, _, g = load_case("spot")
    spec = spec_from_workload(fm, wl)
    assert spec.npairs == 40
    emu = Emu(fm.to_blob(), spec, fm.nq, fm.nv)
    B = 3
    q = np.tile(fm.key("home"), (B, 1))   # feet 3.5 mm inside the floor (sphere radius 0.036 at height 0.0325): d <= d_min, h = relaxation = 0
    frames = task_frames(wl, fm)
    poses, com, _ = emu.fk(q, frames)
    ft = poses.astype(np.float64).copy()
    ft[:, :, 6] += 0.2         # at penetration the witness-point normal points INTO the floor (collision_avoidance_limit.py:49
                               # normalises fromto as it comes), so it is the upward move that all 40 rows oppose
    pk, Gc, hc = emu.fk_jac(q, ft, None, com, dt=wl["dt"], prec="mixed", packed=True)
    assert np.isfinite(hc).sum() == 40 * B
    dq, st, it, *_ = emu.solve(q, None, None, None, Gc, hc, wl["dt"], wl["damping"], use_double=1, pk=pk)
    assert (st & 2).all(), st


def test_degenerate_contact_sets_are_solved_not_flagged():
    """ALOHA with its 1 104-pair collision limit, configurations sampled around the keyframe: a few per cent of them have 8-16
    pairs at the minimum distance between the same two wrist links -- rows that span at most 6 directions, all with h = 0.  The
    general path must solve every one of them (it used to cycle on 4 % and flag them); the optimum of such a wedge is
    ill-conditioned (1e-8 on h moves dq by 1e-4), so the comparison with the oracle allows rare outliers."""
    from oracle import ikoracle
    from mink_b200.workloads import make_inputs, task_frames
    wl, fm, spec, g, emu = _emu("aloha_coll")
    orc = ikoracle.Oracle(fm.to_blob(), spec, fm.nq, fm.nv)
    frames = task_frames(wl, fm)
    B = 768
    inp = make_inputs(fm, wl, B, lambda qq: orc.fk(qq, frames), seed=1000)
    dq_ref, _, st_ref, _ = orc.step(inp["q"], inp["frame_targets"], inp["posture_target"], None, dt=wl["dt"], damping=wl["damping"],
                                    nsteps=1, integrate=False)
    J, e, ep, Gc, hc = emu.fk_jac(inp["q"], inp["frame_targets"], inp["posture_target"], None, dt=wl["dt"], prec="f64")
    assert ((hc == 0).sum(axis=1) >= 8).sum() >= 10      # the sample does contain such contact sets
    dq, st, it, *_ = emu.solve(inp["q"], J, e, ep, Gc, hc, wl["dt"], wl["damping"], use_double=True, io64=True)
    assert not st_ref.any() and not st.any(), np.unique(st, return_counts=True)
    err = np.abs(dq - dq_ref).max(axis=1)
    print("aloha_coll sample: max err %.2e, instances above 1e-6: %d of %d, iterations mean %.1f max %d" % (err.max(), (err > 1e-6).sum(), B, it.mean(), it.max()))
    assert (err > 1e-6).mean() < 0.01 and err.max() < 2e-3


def test_more_finite_rows_than_the_row_window_are_flagged():
    """The general path gathers the pairs inside the detection distance into a window of K2_ROW_WINDOW (64) rows per problem.
    With the detection distance blown up to 10 m every one of ALOHA's 1 104 pairs is finite: the instance must come back
    flagged (BIK_STATUS_QP_MAXITER), not solved on a truncated row set."""
    from mink_b200._abi import spec_from_workload
    from mink_b200.workloads import WORKLOADS

    wl = dict(WORKLOADS["aloha_coll"])
    wl["limits"] = [dict(l, detection_distance=10.0) if l["kind"] == "collision" else l for l in wl["limits"]]
    _, fm, _, g = load_case("aloha_coll")
    spec = spec_from_workload(fm, wl)
    emu = Emu(fm.to_blob(), spec, fm.nq, fm.nv)
    q = g["q"][:2]
    J, e, ep, Gc, hc = emu.fk_jac(q, g["frame_targets"][:2], g["posture_target"], None, dt=wl["dt"], prec="f64")
    assert (np.isfinite(hc).sum(axis=1) > 64).all()
    dq, st, *_ = emu.solve(q, J, e, ep, Gc, hc, wl["dt"], wl["damping"], use_double=True, io64=True)
    assert (st & 2).all(), st
