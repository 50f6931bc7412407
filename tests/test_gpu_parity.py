"""GPU parity: the CUDA path (through the C ABI) against the golden vectors and the C oracle.

Tolerance: BASELINE.json north_star -- dq within 1e-4 rad of the fp64 reference on identical inputs.
  * fp64 entry points (double buffers, what a single numpy Configuration takes): every configuration, the
    ill-conditioned ones included, against the goldens at 1e-6 or tighter;
  * fp32 entry points (the batched fast path): against the goldens at 1e-4, except Spot / edge whose goldens were
    generated from fp64 inputs -- rounding q to fp32 alone moves Spot's optimum by up to ~3e-4 (cost / (2 sqrt(damping))
    = 3e3 times 1e-7) -- so those two are held to 1e-4 against the oracle evaluated on the SAME fp32-rounded inputs
    (test_fp32_entry_points_match_oracle_on_identical_inputs) and to 1e-3 against the fp64-input golden.
Property tests cover BASELINE's full sizes.
"""

import os

import numpy as np
import pytest

torch = pytest.importorskip("torch")
pytestmark = pytest.mark.gpu

from mink_b200._abi import spec_from_workload  # noqa: E402
from mink_b200.workloads import WORKLOADS, make_inputs  # noqa: E402
from tests.helpers import load_case, load_flat, quat_align, task_frames  # noqa: E402

CASES = ["ur5e", "ur5e_dls", "g1", "shadow", "spot", "g1_rel", "edge", "g1_full", "g1_hands", "ur5e_damp", "ur5e_wall",
         "iiwa", "h1", "go1", "stretch", "tidybot", "aloha", "aloha_coll", "leap"]   # the last eight: the reference's other example robots


def _need_gpu():
    if not torch.cuda.is_available():
        pytest.skip("no CUDA device")


def _r32(a):
    """fp32-representable copy of an fp64 array (None passes through)."""
    return None if a is None else np.asarray(a, np.float32).astype(np.float64)


def _engine(name, env=None):
    _need_gpu()
    from mink_b200.engine import DeviceModel, Problem

    old = {}
    for k, v in (env or {}).items():
        old[k] = os.environ.get(k)
        os.environ[k] = str(v)
    try:
        wl, fm, spec, g = load_case(name)
        model = DeviceModel(fm, device=0)
        prob = Problem(model, spec)
    finally:
        for k, v in old.items():
            if v is None:
                os.environ.pop(k, None)
            else:
                os.environ[k] = v
    return wl, fm, spec, g, model, prob


def _oracle(fm, spec):
    from oracle.ikoracle import Oracle

    return Oracle(fm.to_blob(), spec, fm.nq, fm.nv)


def _np(t):
    return t.detach().cpu().numpy().astype(np.float64)


@pytest.mark.parametrize("name", CASES)
def test_fk_and_frame_jacobian(name):
    wl, fm, spec, g, model, prob = _engine(name)
    frames = task_frames(wl, fm)
    poses, com = model.fk(g["q"], frames, want_com=True)
    poses, ref = _np(poses), g["frame_pose"][:, :len(frames)]
    np.testing.assert_allclose(poses[..., 4:], ref[..., 4:], atol=5e-6)
    np.testing.assert_allclose(quat_align(poses[..., :4], ref[..., :4]), ref[..., :4], atol=5e-6)
    if fm.ncom:
        np.testing.assert_allclose(_np(com), g["com"], atol=5e-6)
    np.testing.assert_allclose(_np(model.frame_jacobian(g["q"], frames)), g["J_body"][:, :len(frames)], atol=1e-5)


@pytest.mark.parametrize("name", CASES)
def test_k1_task_errors_and_jacobians(name):
    wl, fm, spec, g, model, prob = _engine(name)
    J, e, ep, Gc, hc = prob.fk_jac(g["q"], g["frame_targets"], g["posture_target"], g.get("com_target"), dt=float(g["dt"]))
    J, e, ep, Gc, hc = map(_np, (J, e, ep, Gc, hc))
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
def test_k2_objective_box_and_solve_from_reference_jacobians(name):
    """K2 alone, fed with the reference's own (J, e) cast to fp32."""
    wl, fm, spec, g, model, prob = _engine(name)
    B, F = g["q"].shape[0], spec.nframe
    f32 = lambda a: torch.tensor(np.ascontiguousarray(a), dtype=torch.float32, device="cuda:0")
    J = f32(np.concatenate([g["J_frame"].reshape(B, 6 * F, fm.nv)] + ([g["J_com"]] if spec.ncom else []), axis=1))
    e = f32(np.concatenate([g["e_frame"].reshape(B, 6 * F)] + ([g["e_com"]] if spec.ncom else []), axis=1))
    ep = f32(g["e_posture"][:, None, :]) if spec.nposture else torch.zeros((B, 0, fm.nv), device="cuda:0")
    Gc = f32(g["G"][:, -spec.npairs:]) if spec.npairs else torch.zeros((B, 0, fm.nv), device="cuda:0")
    hc = f32(g["h"][:, -spec.npairs:]) if spec.npairs else torch.zeros((B, 0), device="cuda:0")
    H, c = prob.objective(J, e, ep, float(g["damping"]))
    scale = np.abs(g["H"]).max()
    np.testing.assert_allclose(_np(H), g["H"], atol=1e-6 * scale)
    np.testing.assert_allclose(_np(c), g["c"], atol=1e-5 * max(1.0, np.abs(g["c"]).max()))
    lo, hi = prob.box(g["q"], float(g["dt"]))
    fin = np.isfinite(g["box_lo"])
    np.testing.assert_allclose(_np(lo)[fin], g["box_lo"][fin], atol=1e-6)
    assert np.all(np.isneginf(_np(lo)[~fin]))
    fin = np.isfinite(g["box_hi"])
    np.testing.assert_allclose(_np(hi)[fin], g["box_hi"][fin], atol=1e-6)
    dq, st = prob.solve(g["q"], J, e, ep, Gc, hc, float(g["dt"]), float(g["damping"]))
    assert int(st.max()) == 0
    np.testing.assert_allclose(_np(dq), g["dq"], atol={"spot": 2e-3, "g1_rel": 5e-5, "aloha_coll": 1e-4}.get(name, 1e-5))   # spot: the fp32 cast of J alone
    # same through the fp64 entry points: the reference's own (J, e) in, the reference's dq out
    f64 = lambda a: torch.tensor(np.ascontiguousarray(a), dtype=torch.float64, device="cuda:0")
    J8 = f64(np.concatenate([g["J_frame"].reshape(B, 6 * F, fm.nv)] + ([g["J_com"]] if spec.ncom else []), axis=1))
    e8 = f64(np.concatenate([g["e_frame"].reshape(B, 6 * F)] + ([g["e_com"]] if spec.ncom else []), axis=1))
    ep8 = f64(g["e_posture"][:, None, :]) if spec.nposture else torch.zeros((B, 0, fm.nv), device="cuda:0", dtype=torch.float64)
    Gc8 = f64(g["G"][:, -spec.npairs:]) if spec.npairs else torch.zeros((B, 0, fm.nv), device="cuda:0", dtype=torch.float64)
    hc8 = f64(g["h"][:, -spec.npairs:]) if spec.npairs else torch.zeros((B, 0), device="cuda:0", dtype=torch.float64)
    H8, c8 = prob.objective(J8, e8, ep8, float(g["damping"]))
    np.testing.assert_allclose(_np(H8), g["H"], atol=1e-8 * scale)      # costs / gains are kept in fp32 (1e-8 relative)
    np.testing.assert_allclose(_np(c8), g["c"], atol=1e-8 * max(1.0, np.abs(g["c"]).max()))
    dq8, st8 = prob.solve(f64(g["q"]), J8, e8, ep8, Gc8, hc8, float(g["dt"]), float(g["damping"]))
    assert int(st8.max()) == 0
    np.testing.assert_allclose(_np(dq8), g["dq"], atol=2e-7 * max(1.0, np.abs(g["dq"]).max()))


@pytest.mark.parametrize("name", CASES)
def test_solve_ik_step_matches_reference(name):
    """The whole step (check_limits -> K1 -> K2 -> integrate) vs reference solve_ik + integrate."""
    wl, fm, spec, g, model, prob = _engine(name)
    q = torch.tensor(g["q"], dtype=torch.float32, device="cuda:0")
    dq, st = prob.step(q, g["frame_targets"], g["posture_target"], g.get("com_target"), dt=float(g["dt"]),
                       damping=float(g["damping"]), nsteps=1, integrate=True)
    assert int(st.max()) == 0
    # spot / edge: fp32 rounding of the golden's fp64 inputs (see the module docstring; the fp64 K1 runs for both);
    # g1_rel: |dq| up to 2.3 rad (no velocity limit) -> relative 1e-4
    tol = {"spot": 1e-3, "g1_rel": 1e-4 * max(1.0, np.abs(g["dq"]).max()), "edge": 1e-3}.get(name, 1e-4)
    err = np.abs(_np(dq) - g["dq"]).max()
    print(f"{name}: max|dq - dq_ref| = {err:.3e}")
    assert err < tol
    np.testing.assert_allclose(_np(q), g["q_next"], atol=2 * tol)


@pytest.mark.parametrize("name", CASES)
def test_rollout_matches_reference(name):
    wl, fm, spec, g, model, prob = _engine(name)
    traj = g["rollout_q"]
    T, RB = traj.shape[0] - 1, traj.shape[1]
    q = torch.tensor(traj[0], dtype=torch.float32, device="cuda:0")
    ct = g["com_target"][:RB] if "com_target" in g else None
    dq, st = prob.step(q, g["frame_targets"][:RB], g["posture_target"], ct, dt=float(g["dt"]), damping=float(g["damping"]),
                       nsteps=T, integrate=True)
    assert int(st.max()) == 0
    np.testing.assert_allclose(_np(q), traj[-1], atol={"spot": 5e-3, "edge": 5e-3, "g1_rel": 2e-3}.get(name, 5e-4))


@pytest.mark.parametrize("name", CASES)
def test_converge_matches_reference(name):
    """bik_converge against the reference's example loop (golden): steps taken, converged flag, final configuration."""
    wl, fm, spec, g, model, prob = _engine(name)
    CB = g["conv_q"].shape[0]
    max_iters, pos, ori = int(g["conv_params"][0]), float(g["conv_params"][1]), float(g["conv_params"][2])
    ct = g["com_target"][:CB] if "com_target" in g else None
    q = torch.tensor(g["q"][:CB], dtype=torch.float32, device="cuda:0")
    it, st = prob.converge(q, g["frame_targets"][:CB], g["posture_target"], ct, dt=float(g["dt"]), damping=float(g["damping"]),
                           max_iters=max_iters, pos_threshold=pos, ori_threshold=ori)
    sti = st.cpu().numpy().astype(np.int64)
    np.testing.assert_array_equal(_np(it), g["conv_iters"])
    np.testing.assert_array_equal((sti & 16) == 0, g["conv_ok"].astype(bool))
    assert int((st & 15).max()) == 0
    np.testing.assert_allclose(_np(q), g["conv_q"], atol={"spot": 1e-2, "edge": 1e-2, "g1_rel": 5e-3}.get(name, 1e-3))


@pytest.mark.parametrize("check_every", [1, 3])
def test_converge_batch_against_oracle(check_every):
    """Per-instance early exit on a ragged UR5e batch: same steps and final q as the oracle's loop; instances that stop early
    keep their configuration; the result does not depend on how often the host polls the device counter."""
    wl, fm, spec, g, model, prob = _engine("ur5e")
    orc = _oracle(fm, spec)
    frames = task_frames(wl, fm)
    B = 1500 + 13
    inp = make_inputs(fm, wl, B, lambda qq: orc.fk(qq, frames), seed=5, sigma=0.05)
    q = torch.tensor(inp["q"], dtype=torch.float32, device="cuda:0")
    it, st = prob.converge(q, inp["frame_targets"], inp["posture_target"], None, dt=wl["dt"], damping=wl["damping"], max_iters=12,
                           pos_threshold=2e-3, ori_threshold=2e-3, check_every=check_every)
    q_ref, it_ref, ok_ref, st_ref = orc.converge(inp["q"], inp["frame_targets"], inp["posture_target"], None, dt=wl["dt"], damping=wl["damping"],
                                                 max_iters=12, pos_threshold=2e-3, ori_threshold=2e-3)
    it = _np(it).astype(np.int32)
    same = it == it_ref
    print(f"converge: iters histogram {np.bincount(it_ref).tolist()} converged {ok_ref.mean():.2f} mismatching iters {int((~same).sum())}/{B}")
    assert same.mean() > 0.995     # an error within fp32 noise of a threshold may flip one decision
    sti = st.cpu().numpy().astype(np.int64)
    np.testing.assert_array_equal(((sti & 16) == 0)[same], ok_ref.astype(bool)[same])
    np.testing.assert_allclose(_np(q)[same], q_ref[same], atol=1e-3)


@pytest.mark.parametrize("group", [1, 2, 4, 8, 16, 32])
def test_every_lane_group_size_against_oracle(group):
    """K1's lanes-per-instance mapping (BIK_K1_GROUP) must not change results; ragged batch (tail tile)."""
    wl, fm, spec, g, model, prob = _engine("g1", env={"BIK_K1_GROUP": group})
    orc = _oracle(fm, spec)
    frames = task_frames(wl, fm)
    B = 263
    inp = make_inputs(fm, wl, B, lambda qq: orc.fk(qq, frames), seed=7)
    J, e, ep, _, _ = prob.fk_jac(inp["q"], inp["frame_targets"], inp["posture_target"], None, dt=wl["dt"])
    Jr, er, epr = orc.fk_jac(inp["q"], inp["frame_targets"], inp["posture_target"], None)
    np.testing.assert_allclose(_np(J), Jr, atol=5e-5)
    np.testing.assert_allclose(_np(e), er, atol=2e-5)
    np.testing.assert_allclose(_np(ep), epr, atol=1e-6)


@pytest.mark.parametrize("env", [{"BIK_USE_TMA": 0}, {"BIK_K2_PATH": "dense"}, {"BIK_K2_PATH": "dense", "BIK_K2_WARPS": 4},
                                 {"BIK_K2_GROUP": 4}, {"BIK_K2_GROUP": 8}, {"BIK_K1_PRECISION": "f64"},
                                 {"BIK_K1_PRECISION": "f64", "BIK_K2_PATH": "dense"}])
def test_alternate_paths(env):
    wl, fm, spec, g, model, prob = _engine("g1", env=env)
    q = torch.tensor(g["q"], dtype=torch.float32, device="cuda:0")
    dq, st = prob.step(q, g["frame_targets"], g["posture_target"], None, dt=float(g["dt"]), damping=float(g["damping"]))
    assert int(st.max()) == 0
    assert np.abs(_np(dq) - g["dq"]).max() < 1e-4


@pytest.mark.parametrize("path", ["dense", "group"])
def test_k2_paths_on_relative_frame_golden(path):
    env = {"BIK_K2_PATH": path}
    wl, fm, spec, g, model, prob = _engine("g1_rel", env=env)
    rep = 5   # 80 instances: more than one tile of every path, ragged tail
    q = torch.tensor(np.tile(g["q"], (rep, 1)), dtype=torch.float32, device="cuda:0")
    dq, st = prob.step(q, np.tile(g["frame_targets"], (rep, 1, 1)), g["posture_target"], None, dt=float(g["dt"]), damping=float(g["damping"]))
    assert int(st.max()) == 0
    tol = 1e-4 * max(1.0, np.abs(g["dq"]).max())
    assert np.abs(_np(dq) - np.tile(g["dq"], (rep, 1))).max() < tol


@pytest.mark.parametrize("name", ["g1", "shadow", "ur5e"])
@pytest.mark.parametrize("path", ["dense", "group", "group4", "k1f64"])
def test_k2_paths_agree_on_a_ragged_batch(name, path):
    """Every K2 path that applies to a box-only problem returns the same optimum (ragged batch: tail tiles of each path);
    "k1f64": the fp64 K1 with its fp64 packed hand-off in front of the default K2."""
    env = {"dense": {"BIK_K2_PATH": "dense"}, "group": {}, "group4": {"BIK_K2_GROUP": 4}, "k1f64": {"BIK_K1_PRECISION": "f64"}}[path]
    wl, fm, spec, g, model, prob = _engine(name, env=env)
    orc = _oracle(fm, spec)
    frames = task_frames(wl, fm)
    B = 1000 + 37
    inp = make_inputs(fm, wl, B, lambda qq: orc.fk(qq, frames), seed=11)
    q = torch.tensor(inp["q"], dtype=torch.float32, device="cuda:0")
    dq, st = prob.step(q, inp["frame_targets"], inp["posture_target"], inp.get("com_target"), dt=wl["dt"], damping=wl["damping"])
    dq_ref, _, st_ref, _ = orc.step(inp["q"], inp["frame_targets"], inp["posture_target"], inp.get("com_target"), dt=wl["dt"],
                                    damping=wl["damping"], nsteps=1, integrate=False)
    assert int(st.max()) == 0 and not st_ref.any()
    err = np.abs(_np(dq) - dq_ref).max()
    print(f"{name}/{path}: max|dq-dq_oracle|={err:.3e}")
    assert err < 1e-4


@pytest.mark.parametrize("env", [{}, {"BIK_K2_SWEEPS": 6}, {"BIK_K2_DYNAMIC": 0}, {"BIK_K2_DYNAMIC": 0, "BIK_K2_GROUP": 4},
                                 {"BIK_K1_GROUP": 8}])
def test_small_group_solver_knobs_against_oracle(env):
    """Elimination of the unbounded dofs, Gauss-Seidel sweeps and tile hand-out only change HOW the optimum of
    mink's QP (solve_ik.py:43-105) is reached: every setting must return the oracle's dq on a ragged G1 batch with active
    bounds, and repeated launches on one stream must keep working (the tile counter rewinds itself)."""
    wl, fm, spec, g, model, prob = _engine("g1", env=env)
    orc = _oracle(fm, spec)
    frames = task_frames(wl, fm)
    B = 3 * 1024 + 5
    inp = make_inputs(fm, wl, B, lambda qq: orc.fk(qq, frames), seed=23)
    dq_ref, _, st_ref, nact = orc.step(inp["q"], inp["frame_targets"], inp["posture_target"], None, dt=wl["dt"], damping=wl["damping"],
                                       nsteps=1, integrate=False)
    assert not st_ref.any() and nact.mean() > 3
    q = torch.tensor(inp["q"], dtype=torch.float32, device="cuda:0")
    for rep in range(3):
        dq, st = prob.step(q, inp["frame_targets"], inp["posture_target"], None, dt=wl["dt"], damping=wl["damping"])
        assert int(st.max()) == 0
        assert np.abs(_np(dq) - dq_ref).max() < 1e-4


@pytest.mark.parametrize("name,B,T", [("g1", 4096 + 3, 8), ("g1_hands", 1024 + 1, 6), ("shadow", 2048, 6)])
def test_rollout_batch_converges_and_matches_oracle(name, B, T):
    """solve_ik + integrate with targets held (examples/humanoid_g1.py:81-94) on a batch: after the first step block
    pivoting alone stalls on a few instances per thousand, so the small-group path carries the previous dq into a
    Gauss-Seidel guess + primal active-set method.  No instance may be flagged, and the trajectory must follow the exact
    oracle's (fp64 state; the device integrates q in fp32, hence the looser bound on q)."""
    wl, fm, spec, g, model, prob = _engine(name)
    orc = _oracle(fm, spec)
    frames = task_frames(wl, fm)
    inp = make_inputs(fm, wl, B, lambda qq: orc.fk(qq, frames), seed=29)
    q = torch.tensor(inp["q"], dtype=torch.float32, device="cuda:0")
    dq, st = prob.step(q, inp["frame_targets"], inp["posture_target"], None, dt=wl["dt"], damping=wl["damping"], nsteps=T, integrate=True)
    assert int(st.max()) == 0, f"{int((st != 0).sum())} instances flagged in a {T}-step rollout"
    dq_ref, q_end, st_ref, _ = orc.step(inp["q"], inp["frame_targets"], inp["posture_target"], None, dt=wl["dt"], damping=wl["damping"],
                                        nsteps=T, integrate=True)
    assert not st_ref.any()
    err_q = np.abs(_np(q) - q_end).max()
    err_dq = np.abs(_np(dq) - dq_ref).max()
    print(f"{name}: {T}-step rollout of {B}: max|q - q_oracle| = {err_q:.2e}, last step max|dq - dq_oracle| = {err_dq:.2e}")
    assert err_q < 5e-4 and err_dq < 2e-4


@pytest.mark.parametrize("name,B", [("g1", 4099), ("shadow", 2050), ("ur5e_dls", 4096), ("spot", 1031)])
def test_batch_against_oracle(name, B):
    wl, fm, spec, g, model, prob = _engine(name)
    orc = _oracle(fm, spec)
    frames = task_frames(wl, fm)
    inp = make_inputs(fm, wl, B, lambda qq: orc.fk(qq, frames), seed=3)
    q = torch.tensor(inp["q"], dtype=torch.float32, device="cuda:0")
    dq, st = prob.step(q, inp["frame_targets"], inp["posture_target"], inp.get("com_target"), dt=wl["dt"], damping=wl["damping"],
                       nsteps=1, integrate=True)
    dq_ref, q_ref, st_ref, nact = orc.step(inp["q"], inp["frame_targets"], inp["posture_target"], inp.get("com_target"), dt=wl["dt"],
                                            damping=wl["damping"], nsteps=1, integrate=True)
    assert int(st.max()) == 0 and not st_ref.any()
    err = np.abs(_np(dq) - dq_ref).max(axis=1)
    print(f"{name}: B={B} max|dq-dq_oracle|={err.max():.3e} median={np.median(err):.3e} active mean={nact.mean():.1f} max={nact.max()}")
    assert err.max() < (1e-4 if name != "spot" else 1e-3)   # spot: the oracle sees the fp64 inputs, the device their fp32 rounding
    np.testing.assert_allclose(_np(q), q_ref, atol=2e-4 if name != "spot" else 2e-3)


def test_full_size_properties_g1():
    """BASELINE config 3 at full size (65 536 instances): size-independent properties."""
    wl, fm, spec, g, model, prob = _engine("g1")
    frames = task_frames(wl, fm)

    def fk(qq):
        p, c = model.fk(qq, frames, want_com=False)
        return _np(p), None

    B = 65536
    inp = make_inputs(fm, wl, B, fk, seed=11)
    q0 = torch.tensor(inp["q"], dtype=torch.float32, device="cuda:0")
    ft = torch.tensor(inp["frame_targets"], dtype=torch.float32, device="cuda:0")
    q = q0.clone()
    dq, st = prob.step(q, ft, inp["posture_target"], None, dt=wl["dt"], damping=wl["damping"], nsteps=1, integrate=False)
    assert int(st.max()) == 0
    assert torch.isfinite(dq).all()
    # (1) feasibility: dq inside the box of configuration + velocity limits
    lo, hi = prob.box(q0, wl["dt"])
    assert bool(((dq >= lo - 1e-6) & (dq <= hi + 1e-6)).all())
    # (2) KKT of the box QP in fp64 from the library's own H, c: projected gradient vanishes
    J, e, ep, Gc, hc = prob.fk_jac(q0, ft, inp["posture_target"], None, dt=wl["dt"])
    H, c = prob.objective(J, e, ep, wl["damping"])
    x = dq.double()
    grad = torch.einsum("bij,bj->bi", H, x) + c
    at_lo = (x <= lo.double() + 1e-6)
    at_hi = (x >= hi.double() - 1e-6)
    free = ~(at_lo | at_hi)
    scale = H.abs().amax(dim=(1, 2)).unsqueeze(1) * 1e-6 + 1e-4
    assert bool((grad.abs()[free] <= scale.expand_as(grad)[free]).all())
    assert bool((grad[at_lo & ~at_hi] >= -scale.expand_as(grad)[at_lo & ~at_hi]).all())
    assert bool((grad[at_hi & ~at_lo] <= scale.expand_as(grad)[at_hi & ~at_lo]).all())
    # (3) determinism
    dq2, _ = prob.step(q0.clone(), ft, inp["posture_target"], None, dt=wl["dt"], damping=wl["damping"])
    assert torch.equal(dq, dq2)
    # (4) fixed point: targets at the current pose and posture target = q  =>  dq = 0
    poses, _ = model.fk(q0, frames)
    dq3, _ = prob.step(q0.clone(), poses, q0.unsqueeze(1), None, dt=wl["dt"], damping=wl["damping"])
    assert float(dq3.abs().max()) < 2e-5
    # (5) integrate keeps the free-joint quaternion on the unit sphere and moves scalar joints by dq
    q1 = q0.clone()
    model.integrate(q1, dq)
    assert float((q1[:, 3:7].norm(dim=1) - 1).abs().max()) < 1e-5
    np.testing.assert_allclose(_np(q1[:, 7:] - q0[:, 7:]), _np(dq[:, 6:]), atol=1e-6)


def test_task_at_target_gives_zero_velocity_ur5e():
    """reference tests/test_solve_ik.py:79-93."""
    wl, fm, spec, g, model, prob = _engine("ur5e")
    frames = task_frames(wl, fm)
    q = torch.tensor(np.tile(fm.key("home"), (5, 1)), dtype=torch.float32, device="cuda:0")
    poses, _ = model.fk(q, frames)
    dq, st = prob.step(q, poses, fm.key("home"), None, dt=wl["dt"], damping=wl["damping"])
    assert float(dq.abs().max()) < 1e-6


def test_out_of_limits_sets_status_flag():
    wl, fm, spec, g, model, prob = _engine("ur5e")
    q = torch.tensor(g["q"], dtype=torch.float32, device="cuda:0")
    q[2, 1] = 100.0
    dq, st = prob.step(q, g["frame_targets"], g["posture_target"], None, dt=wl["dt"], damping=wl["damping"])
    st = st.cpu().numpy()
    assert st[2] & 1 and not (np.delete(st, 2) & 1).any()
    assert (model.check_limits(q).cpu().numpy() != 0).sum() == 1


def test_step_host_entry_point():
    wl, fm, spec, g, model, prob = _engine("g1")
    dq, st, q, up, down = prob.step_host(g["q"], g["frame_targets"], g["posture_target"], None, dt=float(g["dt"]),
                                         damping=float(g["damping"]), nsteps=1, integrate=True)
    assert not st.any()
    assert np.abs(dq - g["dq"]).max() < 1e-4
    np.testing.assert_allclose(q, g["q_next"], atol=2e-4)
    B = g["q"].shape[0]
    assert up == 4 * (B * fm.nq + B * 3 * 7 + fm.nq) and down == 4 * (B * fm.nv + B * fm.nq + B)


def test_step_host_chunking_does_not_change_results():
    """bik_step_host cuts a large batch into chunks on two streams (copies overlap kernels): same dq, q and status as one chunk,
    and as the device-buffer entry point; ragged batch so that the last chunk is partial."""
    wl, fm, spec, g, model, prob = _engine("g1")
    B = 40000 + 77
    rng = np.random.default_rng(2)
    idx = rng.integers(0, g["q"].shape[0], size=B)
    q0 = g["q"][idx].astype(np.float32); ft = g["frame_targets"][idx].astype(np.float32)
    outs = []
    for chunks in (1, 4, 7):
        os.environ["BIK_HOST_CHUNKS"] = str(chunks)
        try:
            dq, st, q, up, down = prob.step_host(q0.copy(), ft, g["posture_target"], None, dt=float(g["dt"]), damping=float(g["damping"]),
                                                 nsteps=1, integrate=True)
        finally:
            os.environ.pop("BIK_HOST_CHUNKS", None)
        assert not st.any()
        outs.append((dq.copy(), q.copy()))
        assert up == 4 * (B * fm.nq + B * 3 * 7 + fm.nq) and down == 4 * (B * fm.nv + B * fm.nq + B)
    for dq, q in outs[1:]:
        np.testing.assert_array_equal(dq, outs[0][0])
        np.testing.assert_array_equal(q, outs[0][1])
    assert np.abs(outs[0][0] - g["dq"][idx]).max() < 1e-4


def test_describe_names_the_mapping():
    wl, fm, spec, g, model, prob = _engine("g1")
    d = prob.describe(float(g["damping"]))
    assert "13/38 nodes visited, f32" in d and "coupled=18" in d and "small-group G=8" in d and d.endswith("f64")
    wl, fm, spec, g, model, prob = _engine("spot")
    d = prob.describe(float(g["damping"]))
    assert "general warp-per-problem" in d and "nodes visited, f64" in d     # ill-conditioned / collision rows: fp64 K1
    wl, fm, spec, g, model, prob = _engine("g1_full")
    assert "small-group G=8 (64-bit masks)" in prob.describe(float(g["damping"]))


def test_empty_batch_and_missing_target():
    wl, fm, spec, g, model, prob = _engine("g1")
    from mink_b200._lib import BikError

    q = torch.zeros((0, fm.nq), dtype=torch.float32, device="cuda:0")
    dq, st = prob.step(q, torch.zeros((0, 3, 7), device="cuda:0"), g["posture_target"], None, dt=0.01)
    assert dq.shape == (0, fm.nv)
    with pytest.raises((BikError, ValueError)):
        prob.step(torch.zeros((2, fm.nq), device="cuda:0"), None, g["posture_target"], None)


# ---- fp64 entry points: the reference's precision ---------------------------------------------------------------------
@pytest.mark.parametrize("name", CASES)
def test_fp64_entry_points_reproduce_the_reference(name):
    """bik_fk_jac64 / bik_step64 (fp64 kernels on the fp64 kinematic constants) against the goldens: FK-derived quantities
    to 1e-9, dq to 2e-7 rad (bounds are kept in fp32), the integrated q and the 8-step rollout -- every BASELINE
    configuration, Spot (cost 200 against damping 1e-3, collision rows) included."""
    wl, fm, spec, g, model, prob = _engine(name)
    f64 = lambda a: None if a is None else torch.tensor(np.ascontiguousarray(a), dtype=torch.float64, device="cuda:0")
    q, ft, pt, ct = f64(g["q"]), f64(g["frame_targets"]), f64(g["posture_target"]), f64(g.get("com_target"))
    J, e, ep, Gc, hc = map(_np, prob.fk_jac(q, ft, pt, ct, dt=float(g["dt"])))
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
    qs = q.clone()
    dq, st = prob.step(qs, ft, pt, ct, dt=float(g["dt"]), damping=float(g["damping"]), nsteps=1, integrate=True)
    assert int(st.max()) == 0 and dq.dtype == torch.float64
    err = np.abs(_np(dq) - g["dq"]).max()
    print(f"{name}: fp64 max|dq - dq_ref| = {err:.3e}")
    assert err < 2e-7 * max(1.0, np.abs(g["dq"]).max())
    np.testing.assert_allclose(_np(qs), g["q_next"], atol=1e-6)
    traj = g["rollout_q"]
    T, RB = traj.shape[0] - 1, traj.shape[1]
    qr = f64(traj[0])
    dq, st = prob.step(qr, ft[:RB], pt, None if ct is None else ct[:RB], dt=float(g["dt"]), damping=float(g["damping"]), nsteps=T, integrate=True)
    assert int(st.max()) == 0
    np.testing.assert_allclose(_np(qr), traj[-1], atol=1e-5)


@pytest.mark.parametrize("name", CASES)
def test_fp32_entry_points_match_oracle_on_identical_inputs(name):
    """The batched fp32 fast path against the oracle evaluated on the SAME fp32-representable inputs (north_star:
    identical inputs): every configuration within 1e-4 rad -- the ill-conditioned ones because bik_step switches K1
    and the hand-off to fp64 by itself (bik_problem_describe says so)."""
    wl, fm, spec, g, model, prob = _engine(name)
    orc = _oracle(fm, spec)
    q, ft, pt, ct = _r32(g["q"]), _r32(g["frame_targets"]), _r32(g["posture_target"]), _r32(g.get("com_target"))
    dq_ref, q_ref, st_ref, _ = orc.step(q, ft, pt, ct, dt=float(g["dt"]), damping=float(g["damping"]), nsteps=1, integrate=True)
    qd = torch.tensor(q, dtype=torch.float32, device="cuda:0")
    dq, st = prob.step(qd, ft, pt, ct, dt=float(g["dt"]), damping=float(g["damping"]), nsteps=1, integrate=True)
    assert int(st.max()) == 0 and not st_ref.any()
    err = np.abs(_np(dq) - dq_ref).max()
    print(f"{name}: fp32 entry, identical inputs: max|dq - dq_oracle| = {err:.3e}")
    assert err < 1e-4 * max(1.0, np.abs(dq_ref).max())
    np.testing.assert_allclose(_np(qd), q_ref, atol=2e-4 * max(1.0, np.abs(dq_ref).max()))


def test_inconsistent_limits_set_the_infeasible_flag():
    """A dof 1 rad past its limit under a velocity limit: the reference's QP is infeasible (qpsolvers returns None,
    solve_ik.py:103 asserts).  Device: BIK_STATUS_QP_INFEASIBLE on that instance only, on both K2 paths."""
    for env in ({}, {"BIK_K2_PATH": "dense"}):
        wl, fm, spec, g, model, prob = _engine("g1", env=env)
        orc = _oracle(fm, spec)
        q = g["q"][:5].copy()
        d = 20
        q[3, int(fm.dof_qadr[d])] = fm.dof_hi[d] + 1.0
        qd = torch.tensor(q, dtype=torch.float32, device="cuda:0")
        dq, st = prob.step(qd, g["frame_targets"][:5], g["posture_target"], None, dt=float(g["dt"]), damping=float(g["damping"]))
        st = st.cpu().numpy()
        _, _, st_ref, _ = orc.step(q, g["frame_targets"][:5], g["posture_target"], None, dt=float(g["dt"]), damping=float(g["damping"]))
        assert st[3] & 8 and st[3] & 1 and not (np.delete(st, 3) & 8).any()
        assert st_ref[3] != 0 and not np.delete(st_ref, 3).any()


@pytest.mark.parametrize("name,B,T", [("spot", 1024 + 7, 12), ("g1_full", 1024 + 5, 10)])
def test_general_and_wide_paths_in_rollouts(name, B, T):
    """Rollouts (targets held, q integrated on the device) on the problems that used to need 10-100 factorisations per
    instance: collision rows (general path: block pivoting with the primal active-set fallback) and the 43 coupled dofs of
    the reference's humanoid example (small-group path with 64-bit masks).  No instance may be flagged; the trajectory
    follows the oracle's."""
    wl, fm, spec, g, model, prob = _engine(name)
    orc = _oracle(fm, spec)
    frames = task_frames(wl, fm)
    inp = make_inputs(fm, wl, B, lambda qq: orc.fk(qq, frames), seed=41, sigma=0.05)
    q0, ft, pt, ct = _r32(inp["q"]), _r32(inp["frame_targets"]), _r32(inp["posture_target"]), _r32(inp.get("com_target"))
    q = torch.tensor(q0, dtype=torch.float32, device="cuda:0")
    dq, st = prob.step(q, ft, pt, ct, dt=wl["dt"], damping=wl["damping"], nsteps=T, integrate=True)
    # bit 1 (a joint left its range) is legitimate where the workload has no ConfigurationLimit (Spot): the reference warns
    assert int((st & ~1).max()) == 0, f"{int(((st & ~1) != 0).sum())} instances flagged (bits {np.unique(st.cpu().numpy())})"
    dq_ref, q_end, st_ref, _ = orc.step(q0, ft, pt, ct, dt=wl["dt"], damping=wl["damping"], nsteps=T, integrate=True)
    ok = st_ref == 0
    err_q = np.abs(_np(q) - q_end)[ok].max()
    print(f"{name}: {T}-step rollout of {B}: max|q - q_oracle| = {err_q:.2e} (oracle flagged {int((~ok).sum())})")
    assert err_q < 2e-3
    # iteration statistics of one more step from the reached configuration
    J, e, ep, Gc, hc = prob.fk_jac(q, ft, pt, ct, dt=wl["dt"])
    _, st2, it = prob.solve(q, J, e, ep, Gc, hc, wl["dt"], wl["damping"], return_iters=True)
    it = it.cpu().numpy()
    print(f"{name}: cold-start factorisations at the reached configuration: mean {it.mean():.2f} max {it.max()}")
    assert int(st2.max()) == 0 and it.max() <= 60


def test_converge_device_loop_matches_host_polled_loop():
    """bik_converge runs its loop as a CUDA-graph WHILE node (the condition is set on the device); BIK_CONVERGE_GRAPH=0 is the
    host-polled loop.  Same steps, flags and configurations; a second call with the same buffers reuses the graph, a call with
    other thresholds rebuilds it."""
    wl, fm, spec, g, model, prob = _engine("ur5e")
    orc = _oracle(fm, spec)
    frames = task_frames(wl, fm)
    B = 700 + 9
    inp = make_inputs(fm, wl, B, lambda qq: orc.fk(qq, frames), seed=15, sigma=0.05)
    ft = torch.tensor(inp["frame_targets"], dtype=torch.float32, device="cuda:0")
    pt = torch.tensor(inp["posture_target"], dtype=torch.float32, device="cuda:0")
    q = torch.empty((B, fm.nq), dtype=torch.float32, device="cuda:0")
    out = {}
    for mode, thr in (("1", 2e-3), ("1", 2e-3), ("1", 5e-3), ("0", 2e-3), ("0", 5e-3)):
        os.environ["BIK_CONVERGE_GRAPH"] = mode
        try:
            q.copy_(torch.tensor(inp["q"], dtype=torch.float32))
            it, st = prob.converge(q, ft, pt, None, dt=wl["dt"], damping=wl["damping"], max_iters=10, pos_threshold=thr, ori_threshold=thr,
                                   check_every=2)
        finally:
            os.environ.pop("BIK_CONVERGE_GRAPH", None)
        res = (it.cpu().numpy().copy(), st.cpu().numpy().copy(), q.cpu().numpy().copy())
        if (mode, thr) in out:
            for a, b in zip(out[(mode, thr)], res):
                np.testing.assert_array_equal(a, b)       # replaying the cached graph is deterministic
        out[(mode, thr)] = res
    for thr in (2e-3, 5e-3):
        for a, b in zip(out[("1", thr)], out[("0", thr)]):
            np.testing.assert_array_equal(a, b)
    assert (out[("1", 5e-3)][0] <= out[("1", 2e-3)][0]).all() and (out[("1", 5e-3)][0] < out[("1", 2e-3)][0]).any()


def test_one_problem_used_from_two_streams():
    """The K1 -> K2 hand-off buffers, tile counters and warm start belong to the problem handle: calls issued on different
    streams must not overlap on them (each call waits for the event the previous one recorded)."""
    _need_gpu()
    wl, fm, spec, g, model, prob = _engine("g1")
    orc = _oracle(fm, spec)
    frames = task_frames(wl, fm)
    B = 20000
    sets = [make_inputs(fm, wl, B, lambda qq: orc.fk(qq, frames), seed=s) for s in (21, 22)]
    dev = [dict(q=torch.tensor(i["q"], dtype=torch.float32, device="cuda:0"),
                ft=torch.tensor(i["frame_targets"], dtype=torch.float32, device="cuda:0")) for i in sets]
    ref = []
    for d, i in zip(dev, sets):
        q = d["q"].clone()
        dq, st = prob.step(q, d["ft"], i["posture_target"], None, dt=wl["dt"], damping=wl["damping"], nsteps=3, integrate=True)
        ref.append((_np(dq), _np(q)))
    torch.cuda.synchronize()
    streams = [torch.cuda.Stream(), torch.cuda.Stream()]
    for rep in range(4):
        outs = []
        for s, d, i in zip(streams, dev, sets):
            with torch.cuda.stream(s):
                q = d["q"].clone()
                dq, st = prob.step(q, d["ft"], i["posture_target"], None, dt=wl["dt"], damping=wl["damping"], nsteps=3, integrate=True)
                outs.append((dq, q))
        torch.cuda.synchronize()
        for (dq, q), (dq_ref, q_ref) in zip(outs, ref):
            assert np.array_equal(_np(dq), dq_ref) and np.array_equal(_np(q), q_ref)


def test_degenerate_contact_sets_are_solved_not_flagged():
    """ALOHA with its 1 104-pair collision limit around the keyframe: 8-16 pairs at the minimum distance between the same two
    links give working sets with dependent rows (h = 0).  Every instance must be solved (status 0) and follow the oracle; the
    optimum of such a wedge is ill-conditioned, so rare outliers above 1e-6 are tolerated, none above 2e-3."""
    wl, fm, spec, g, model, prob = _engine("aloha_coll")
    orc = _oracle(fm, spec)
    frames = task_frames(wl, fm)
    B = 1024 + 3
    inp = make_inputs(fm, wl, B, lambda qq: orc.fk(qq, frames), seed=1000)
    dq_ref, _, st_ref, _ = orc.step(inp["q"], inp["frame_targets"], inp["posture_target"], None, dt=wl["dt"], damping=wl["damping"],
                                    nsteps=1, integrate=False)
    q = torch.tensor(inp["q"], dtype=torch.float64, device="cuda:0")
    dq, st = prob.step(q, inp["frame_targets"], inp["posture_target"], None, dt=wl["dt"], damping=wl["damping"], nsteps=1, integrate=False)
    assert not st_ref.any() and int(st.max()) == 0, np.unique(_np(st), return_counts=True)
    err = np.abs(_np(dq) - dq_ref).max(axis=1)
    print(f"aloha_coll sample: max err {err.max():.2e}, above 1e-6: {(err > 1e-6).sum()} of {B}")
    assert (err > 1e-6).mean() < 0.01 and err.max() < 2e-3
