"""Held targets on the device: bik_track_hold / bik_track_hold64 through Problem.track(hold=), and track_ik(hold=).

A NULL or all-zero mask gives what bik_track_coll gives; with random runs the fp64 call is T converge calls in which the held
targets are set from bik_fk64 at the configuration each run starts from; a fully held instance stays put; a held foot does
not drift over its run; the cached converge graph follows the hold buffer; the front end builds the same mask.
"""

import numpy as np
import pytest

torch = pytest.importorskip("torch")
pytestmark = pytest.mark.gpu

from mink_b200._abi import TASK_COM, TASK_FRAME, TASK_POSTURE, TASK_RELATIVE_FRAME  # noqa: E402
from tests.helpers import load_case, qmul_np, qrot_np, track_case  # noqa: E402
from tests.test_gpu_posture_weights import _problem  # noqa: E402
from tests.test_track_hold_cpu import CONV, _runs  # noqa: E402

DT = {np.float32: torch.float32, np.float64: torch.float64}


def _case(name, dtype, B, T, seed):
    if not torch.cuda.is_available():
        pytest.skip("no CUDA device")
    _, fm, spec, _ = load_case(name)
    c = track_case(name, B=B, T=T, seed=seed, dtype=dtype)
    c["fm"], c["spec"], c["prob"] = fm, spec, _problem(fm, spec)
    c["dev"] = lambda a, dt=DT[dtype]: None if a is None else torch.tensor(np.ascontiguousarray(a), dtype=dt, device="cuda:0")
    c["H"] = spec.nframe + spec.ncom + spec.nposture
    c["fr"] = [t for t in spec.tasks if t.kind in (TASK_FRAME, TASK_RELATIVE_FRAME)]
    # every frame-like task's sequence: track_case's for the FRAME tasks, a RELATIVE_FRAME task's pose in its root at q0
    cap0 = _capture(c, c["dev"](c["q0"]))
    cols, i = [], 0
    for k, t in enumerate(c["fr"]):
        if t.kind == TASK_FRAME:
            cols.append(c["ft"][:, :, i]); i += 1
        else:
            cols.append(np.repeat(cap0[k].cpu().numpy()[:, None], T, axis=1))
    c["ft"] = np.ascontiguousarray(np.stack(cols, axis=2))
    c["pt"] = np.repeat(c["pt"], spec.nposture, axis=1)
    c["d"] = dict(ft=c["dev"](c["ft"]), ct=c["dev"](c["ct"]), pt=c["dev"](c["pt"]))
    return c


def _capture(c, q):
    """What each held task captures at q (bik_fk / bik_fk64 on the device; root^-1 * frame composed on the host), in hold-column
    order: [B, 7] per frame-like task, [B, 3] per CoM task, [B, nq] per posture-type task."""
    fr = c["fr"]
    roots = [t.root for t in fr if t.kind == TASK_RELATIVE_FRAME]
    poses, com = c["prob"].model.fk(q, [t.frame for t in fr] + roots, want_com=True)
    out, r = [], len(fr)
    for i, t in enumerate(fr):
        p = poses[:, i]
        if t.kind == TASK_RELATIVE_FRAME:
            pr, pf = poses[:, r].double().cpu().numpy(), p.double().cpu().numpy()
            cj = pr[:, :4] * np.array([1, -1, -1, -1])
            rel = np.concatenate([qmul_np(cj, pf[:, :4]), qrot_np(cj, pf[:, 4:] - pr[:, 4:])], axis=1)
            p, r = torch.tensor(rel, dtype=q.dtype, device=q.device), r + 1
        out.append(p)
    out += [com for t in c["spec"].tasks if t.kind == TASK_COM]
    out += [q.clone() for t in c["spec"].tasks if t.kind == TASK_POSTURE]
    return out


def _track(c, hold, ln=None, prob=None):
    d = c["d"]
    q = c["dev"](c["q0"])
    hd = None if hold is None else torch.as_tensor(np.asarray(hold, np.uint8), device="cuda:0") if isinstance(hold, np.ndarray) else hold
    out = (prob or c["prob"]).track(q, d["ft"], d["pt"], d["ct"], lengths=ln, hold=hd, **c["kw"], **CONV)
    return (q, *out)


def _equal(a, b):
    torch.testing.assert_close(a, b, rtol=0, atol=0, equal_nan=True)


@pytest.mark.parametrize("dtype", [np.float32, np.float64], ids=["f32", "f64"])
@pytest.mark.parametrize("name", ["ur5e", "g1", "edge"])
def test_null_and_zero_masks_are_track_coll(name, dtype):
    """A NULL mask and an all-zero mask both give bik_track_coll's q, q_traj, iters, status and passes, bit for bit."""
    c = _case(name, dtype, B=300 + 3, T=4, seed=3)
    ln = np.random.default_rng(4).integers(0, c["T"] + 1, size=c["B"]).astype(np.int32)
    ref = _track(c, None, ln)
    for hold in (None, np.zeros((c["B"], c["T"], c["H"]), bool)):
        for x, y in zip(_track(c, hold, ln), ref):
            _equal(x, y)


@pytest.mark.parametrize("name", ["edge", "g1"])
def test_fp64_equals_per_frame_loop(name):
    """Random runs: bik_track_hold64 matches T bik_converge_coll64 calls in which, before the first frame of each run, the held
    targets are set from bik_fk64 at the previous frame's result (q_traj within 1e-9, iters and status equal)."""
    c = _case(name, np.float64, B=128, T=8, seed=5)
    B, T, F, Cn = c["B"], c["T"], c["spec"].nframe, c["spec"].ncom
    hold = _runs(np.random.default_rng(6), B, T, c["H"])
    _, q_traj, it, st, _ = _track(c, hold)
    d = c["d"]
    q = c["dev"](c["q0"])
    hmask = torch.as_tensor(hold, device="cuda:0")
    held = None
    for t in range(T):
        start = hmask[:, t] & (~hmask[:, t - 1] if t > 0 else torch.ones_like(hmask[:, t]))
        if bool(start.any()):
            cap = _capture(c, q)
            held = cap if held is None else [torch.where(start[:, k, None], cap[k], held[k]) for k in range(len(cap))]
        ft, ct, pt = d["ft"][:, t].clone(), None if d["ct"] is None else d["ct"][:, t].clone(), d["pt"].clone()
        for k in range(c["H"]):
            on = hmask[:, t, k]
            dst = ft[:, k] if k < F else (ct[:, k - F] if k < F + Cn else pt[:, k - F - Cn])
            dst[on] = held[k][on] if held is not None else dst[on]
        itt, stt = c["prob"].converge(q, ft, pt, ct, **c["kw"], **CONV)
        torch.testing.assert_close(q_traj[:, t], q, rtol=0, atol=1e-9)
        _equal(it[:, t], itt); _equal(st[:, t], stt)


@pytest.mark.parametrize("dtype", [np.float32, np.float64], ids=["f32", "f64"])
def test_everything_held_stays_put(dtype):
    """With every task held on a frame, an instance takes one step and stays where it is: within 1e-12 in fp64, and within
    2e-6 in fp32, where the captured targets' rounding (the pose through bik_fk's quaternion, the CoM summed as bik_fk sums it)
    leaves errors of about 1e-7 that the step follows (1.1e-6 measured on one dof of G1)."""
    c = _case("g1", dtype, B=64, T=5, seed=7)
    hold = np.zeros((c["B"], c["T"], c["H"]), bool)
    hold[::2] = True
    q, q_traj, it, st, _ = _track(c, hold)
    tol = 1e-12 if dtype == np.float64 else 2e-6
    prev = torch.cat([c["dev"](c["q0"])[:, None], q_traj[:, :-1]], dim=1)
    assert bool((it[::2] == 1).all())
    torch.testing.assert_close(q_traj[::2], prev[::2], rtol=0, atol=tol)


@pytest.mark.parametrize("dtype", [np.float32, np.float64], ids=["f32", "f64"])
def test_held_foot_does_not_drift(dtype):
    """G1: each foot is held for alternating 20-frame runs while every other target moves.  On every converged frame of a
    run, the foot's pose from FK of q_traj stays within the thresholds of its pose at the configuration the run began from.
    (The moving targets conflict with the held foot on most frames, more so as the path moves on: the first run's frames
    converge more often.)"""
    c = _case("g1", dtype, B=64, T=40, seed=8)
    B, T = c["B"], c["T"]
    hold = np.zeros((B, T, c["H"]), bool)
    runs = (np.arange(T) // 20) % 2 == 0
    hold[:, :, 0] = runs
    hold[:, :, 1] = ~runs
    q, q_traj, it, st, _ = _track(c, hold)
    q_prev = torch.cat([c["dev"](c["q0"])[:, None], q_traj[:, :-1]], dim=1)
    frames = [c["fr"][0].frame, c["fr"][1].frame]
    pose, _ = c["prob"].model.fk(q_traj.reshape(B * T, -1), frames)
    pose = pose.reshape(B, T, 2, 7).double().cpu().numpy()
    start = pose.copy()
    for f in range(2):
        col = hold[0, :, f]
        for t in range(T):
            if col[t] and (t == 0 or not col[t - 1]):
                p0, _ = c["prob"].model.fk(q_prev[:, t], [frames[f]])
                anchor = p0[:, 0].double().cpu().numpy()
            if col[t]:
                start[:, t, f] = anchor
    ok = ((st & 16) == 0).cpu().numpy()
    assert (hold[:, :, :2] & ok[:, :, None]).sum() >= 50   # converged frames with a foot held
    for f in range(2):
        on = hold[:, :, f] & ok
        if not on.any():
            continue
        dp = np.linalg.norm(pose[:, :, f, 4:] - start[:, :, f, 4:], axis=-1)
        rel = qmul_np((start[:, :, f, :4] * np.array([1, -1, -1, -1])).reshape(-1, 4), pose[:, :, f, :4].reshape(-1, 4))
        ang = (2 * np.arcsin(np.linalg.norm(rel[:, 1:], axis=-1).clip(0, 1))).reshape(B, T)
        assert dp[on].max() <= CONV["pos_threshold"] * 1.01, dp[on].max()
        assert ang[on].max() <= CONV["ori_threshold"] * 1.01, ang[on].max()


def test_cached_graph_follows_the_hold_buffer():
    """Calls alternating between two hold buffers give what a problem without a cached graph gives; so does rewriting a buffer
    in place between two calls (the same buffer reuses the graph)."""
    c = _case("g1", np.float32, B=128, T=4, seed=9)
    rng = np.random.default_rng(10)
    ha = torch.as_tensor(_runs(rng, c["B"], c["T"], c["H"]).astype(np.uint8), device="cuda:0")
    hb = torch.as_tensor(_runs(rng, c["B"], c["T"], c["H"]).astype(np.uint8), device="cuda:0")
    fresh = lambda h: _track(c, h, prob=_problem(c["fm"], c["spec"]))
    ref_a, ref_b, ref_0 = fresh(ha), fresh(hb), fresh(None)
    for h, ref in ((ha, ref_a), (hb, ref_b), (ha, ref_a), (None, ref_0), (hb, ref_b)):
        for x, y in zip(_track(c, h), ref):
            _equal(x, y)
    hb.copy_(ha)
    for x, y in zip(_track(c, hb), ref_a):
        _equal(x, y)


def test_front_end_hold():
    """track_ik(hold={task: mask}) on a float32 batch and on a single fp64 configuration gives what Problem.track(hold=) gives;
    a task held on every frame needs no target; wrong shapes and a DampingTask raise InvalidTarget."""
    import mink_b200 as mink
    from mink_b200.lie import SE3
    from mink_b200.workloads import WORKLOADS

    c = _case("g1", np.float32, B=16, T=6, seed=11)
    wl, fm, B, T = WORKLOADS["g1"], c["fm"], c["B"], c["T"]
    rng = np.random.default_rng(12)
    foot = rng.random((B, T)) < 0.5
    pel = rng.random(T) < 0.5

    def setup(q0):
        cfg = mink.Configuration(fm, q0)
        tasks = [mink.FrameTask(f["name"], f["type"], f["position_cost"], f["orientation_cost"], lm_damping=f["lm_damping"])
                 for f in wl["frames"]]
        post = mink.PostureTask(fm, cost=wl["posture"]["cost"])
        post.set_target(np.asarray(c["q0"][0], np.float64))
        limits = [mink.ConfigurationLimit(fm),
                  mink.VelocityLimit(fm, {n: np.pi for n, t in zip(fm.names["joint"], fm.node_type) if t >= 2})]
        return cfg, tasks + [post], limits

    ft = c["ft"].astype(np.float64)
    for f64 in (False, True):
        if f64:
            b = 3
            q0 = np.asarray(c["q0"][b], np.float64)
            cfg, tasks, limits = setup(q0.copy())
            targets = {tasks[0]: ft[b, :, 0], tasks[1]: SE3(ft[b, :, 1]), tasks[2]: ft[b, :, 2]}
            hold = {tasks[0]: foot[b], tasks[2]: pel, tasks[3]: np.ones(T, bool)}
            qd = torch.tensor(q0[None], dtype=torch.float64, device="cuda:0")
            ftd = torch.tensor(ft[b:b + 1], dtype=torch.float64, device="cuda:0")
            mask = np.stack([foot[b], np.zeros(T, bool), pel, np.ones(T, bool)], axis=-1)[None]
        else:
            q0 = torch.tensor(c["q0"], dtype=torch.float32, device="cuda:0")
            cfg, tasks, limits = setup(q0.clone())
            targets = {tasks[0]: c["d"]["ft"][:, :, 0], tasks[1]: c["d"]["ft"][:, :, 1], tasks[2]: c["d"]["ft"][:, :, 2]}
            hold = {tasks[0]: foot, tasks[2]: pel}
            qd, ftd = q0.clone(), c["d"]["ft"]
            mask = np.stack([foot, np.zeros((B, T), bool), np.broadcast_to(pel, (B, T)), np.zeros((B, T), bool)], axis=-1)
        q_traj, iters, ok = mink.track_ik(cfg, tasks, c["kw"]["dt"], targets, damping=c["kw"]["damping"], limits=limits, hold=hold, **CONV)
        from mink_b200.ik import _problem as ik_problem
        prob, _ = ik_problem(cfg, tasks, limits)
        pt = torch.tensor(np.asarray(tasks[3].target_q, np.float64).reshape(1, 1, -1), dtype=qd.dtype, device="cuda:0")
        r_traj, r_it, r_st, _ = prob.track(qd, ftd, pt, None, dt=c["kw"]["dt"], damping=c["kw"]["damping"],
                                           hold=torch.as_tensor(mask.astype(np.uint8), device="cuda:0"), **CONV)
        if f64:
            np.testing.assert_array_equal(q_traj, r_traj[0].cpu().numpy())
            np.testing.assert_array_equal(iters, r_it[0].cpu().numpy())
        else:
            _equal(q_traj, r_traj); _equal(iters, r_it)

    cfg, tasks, limits = setup(torch.tensor(c["q0"], dtype=torch.float32, device="cuda:0"))
    tasks[2].transform_target_to_world = None   # held on every frame: no target needed
    mink.track_ik(cfg, tasks, 1e-2, {tasks[0]: ft[:, :, 0], tasks[1]: ft[:, :, 1]}, limits=limits,
                  hold={tasks[2]: np.ones(T, bool)}, **CONV)
    with pytest.raises(mink.TargetNotSet):   # held on some frames only: its other frames need a target
        mink.track_ik(cfg, tasks, 1e-2, {tasks[0]: ft[:, :, 0], tasks[1]: ft[:, :, 1]}, limits=limits, hold={tasks[2]: pel}, **CONV)
    damp = mink.DampingTask(fm, cost=0.1)
    feet = {tasks[0]: ft[:, :, 0], tasks[1]: ft[:, :, 1], tasks[2]: ft[:, :, 2]}
    for bad in ({damp: np.ones(T, bool)}, {tasks[0]: np.ones(T + 1, bool)}, {tasks[0]: np.ones((B + 1, T), bool)},
                {tasks[0]: np.ones((B, T, 1), bool)}):
        with pytest.raises(mink.InvalidTarget):
            mink.track_ik(cfg, tasks + [damp], 1e-2, feet, limits=limits, hold=bad, **CONV)
