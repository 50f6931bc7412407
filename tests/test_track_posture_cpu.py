"""bik_track with a posture target sequence (bik_inputs.posture_batched = 2 or 3), on the kernel headers compiled for the host
(tests/host_emu/emu_posture.cpp), no GPU needed.

The definition: for every instance b, bik_track with a posture sequence equals bik_converge called on frames 0..lengths[b]-1
in turn, frame t's call with frame t's posture target as an ordinary (form 0 / 1) target.  K1 copies frame t's posture rows
into a per-instance buffer on the frame's first pass and K2 reads that buffer, so the emulated loops must agree bit for bit.
"""

import numpy as np
import pytest

from mink_b200.workloads import WORKLOADS

CONV = dict(max_iters=10, pos_threshold=2e-3, ori_threshold=2e-3)


def _case(name, dtype, B=64 + 5, T=6, seed=12, wl=None):
    """As tests.helpers.track_case (targets from the oracle's FK along a seeded joint path), for workload `name` or the
    workload dict `wl`, plus a joint-space sequence pseq [B, T, P, nq]: every hinge / slide of each instance's posture target
    drifts away from q0 by a random walk (free-joint and ball coordinates stay at q0's, so quaternions stay normalised)."""
    from mink_b200._abi import spec_from_workload
    from mink_b200.workloads import load_flat, make_inputs, task_frames
    from oracle.ikoracle import Oracle
    from tests.emu_posture_lib import PostureEmu

    wl = wl or WORKLOADS[name]
    fm = load_flat(wl["robot"])
    spec = spec_from_workload(fm, wl)
    emu = PostureEmu(fm.to_blob(), spec, fm.nq, fm.nv)
    orc = Oracle(fm.to_blob(), spec, fm.nq, fm.nv)
    frames = task_frames(wl, fm)
    inp = make_inputs(fm, wl, B, lambda qq: orc.fk(qq, frames), seed=seed, sigma=0.3)
    rng = np.random.default_rng(seed + 1)
    path = np.repeat(inp["q"][:, None, :], T, axis=1)
    seq = np.repeat(inp["q"][:, None, None, :], T, axis=1).repeat(spec.nposture, axis=2)
    frac = np.arange(1, T + 1) / T
    for n in range(fm.nnode):
        if int(fm.node_type[n]) >= 2:   # hinge / slide
            a = int(fm.node_qadr[n])
            path[:, :, a] += rng.normal(0.0, 0.3, size=B)[:, None] * frac[None, :]
            seq[:, :, :, a] += np.cumsum(rng.normal(0.0, 0.05, size=(B, T, spec.nposture)), axis=1)
    poses, com = orc.fk(path.reshape(B * T, fm.nq), frames)
    ft = np.asarray(poses, dtype).reshape(B, T, -1, 7)
    ct = np.asarray(com, dtype).reshape(B, T, -1, 3) if spec.ncom else None
    return dict(emu=emu, orc=orc, q0=inp["q"].astype(dtype), ft=ft, ct=ct, pseq=seq.astype(dtype),
                kw=dict(dt=wl["dt"], damping=wl["damping"]), B=B, T=T)


def _per_frame(c, pts):
    """The definition's loop: one emulated converge per frame on the same q; pts(t) is frame t's posture target."""
    B, T, nq = c["B"], c["T"], c["q0"].shape[1]
    q = c["q0"]
    q_loop, it_loop, st_loop = np.zeros((B, T, nq), q.dtype), np.zeros((B, T), np.int32), np.zeros((B, T), np.int32)
    for t in range(T):
        q, it_loop[:, t], st_loop[:, t] = c["emu"].converge(q, c["ft"][:, t], pts(t), None if c["ct"] is None else c["ct"][:, t],
                                                            **c["kw"], **CONV)
        q_loop[:, t] = q
    return q_loop, it_loop, st_loop


def _check_equal(c, loop, out, lengths):
    q_loop, it_loop, st_loop = loop
    q_end, q_traj, it, st, passes = out
    B, T = c["B"], c["T"]
    has = np.arange(T)[None, :] < lengths[:, None]
    np.testing.assert_array_equal(q_traj[has], q_loop[has])
    np.testing.assert_array_equal(it[has], it_loop[has])
    np.testing.assert_array_equal(st[has], st_loop[has])
    assert np.isnan(q_traj[~has]).all() and (it[~has] == -1).all() and (st[~has] == -1).all()
    q_ref = np.where(lengths[:, None] > 0, q_loop[np.arange(B), np.maximum(lengths - 1, 0)], c["q0"])
    np.testing.assert_array_equal(q_end, q_ref)
    assert passes == int(np.where(has, it + 1, 0).sum(1).max())


def _lengths(c):
    ln = np.random.default_rng(2).integers(0, c["T"] + 1, size=c["B"]).astype(np.int32)
    ln[:3] = [0, c["T"], 1]
    return ln


@pytest.mark.parametrize("dtype", [np.float32, np.float64], ids=["f32", "f64"])
@pytest.mark.parametrize("name", ["ur5e", "h1", "tidybot", "ur5e_wall"])
def test_sequence_equals_per_frame_converge(name, dtype):
    """ur5e: small-group K2; h1: CoM sequence too; tidybot: per-dof posture cost with zeros; ur5e_wall: collision rows, so the
    fp64 K1 (also for fp32 callers) and the general K2.  Form 3 against per-instance targets, form 2 against a shared one."""
    c = _case(name, dtype)
    ln = _lengths(c)
    seq = c["pseq"]
    loop = _per_frame(c, lambda t: seq[:, t])
    out = c["emu"].track(c["q0"], c["ft"], seq, c["ct"], **c["kw"], **CONV, lengths=ln, posture_form=3)
    _check_equal(c, loop, out, ln)
    shared = seq[7]   # [T, P, nq]: instance 7's sequence for everybody
    loop2 = _per_frame(c, lambda t: shared[t][None])
    out2 = c["emu"].track(c["q0"], c["ft"], shared, c["ct"], **c["kw"], **CONV, lengths=ln, posture_form=2)
    _check_equal(c, loop2, out2, ln)
    assert not np.array_equal(out[1][ln > 1], out2[1][ln > 1])   # the two sequences do steer the instances apart


@pytest.mark.parametrize("dtype", [np.float32, np.float64], ids=["f32", "f64"])
def test_sequence_spot(dtype):
    """Spot (the fp64 K1 for fp32 callers by the conditioning estimate) with a PostureTask added to its workload."""
    c = _case("spot", dtype, B=32 + 3, T=5, wl=dict(WORKLOADS["spot"], posture=dict(cost=1e-2)))
    ln = _lengths(c)
    loop = _per_frame(c, lambda t: c["pseq"][:, t])
    out = c["emu"].track(c["q0"], c["ft"], c["pseq"], c["ct"], **c["kw"], **CONV, lengths=ln, posture_form=3)
    _check_equal(c, loop, out, ln)


@pytest.mark.parametrize("dtype", [np.float32, np.float64], ids=["f32", "f64"])
def test_constant_sequence_equals_held_target(dtype):
    """A sequence that repeats one target gives what the call without a sequence gives, bit for bit (forms 3 / 1, 2 / 0)."""
    c = _case("ur5e", dtype, seed=5)
    ln = _lengths(c)
    T = c["T"]
    held = c["pseq"][:, 2]                                        # [B, P, nq]
    a = c["emu"].track(c["q0"], c["ft"], held, None, **c["kw"], **CONV, lengths=ln)
    b = c["emu"].track(c["q0"], c["ft"], np.repeat(held[:, None], T, axis=1), None, **c["kw"], **CONV, lengths=ln, posture_form=3)
    for x, y in zip(a, b):
        np.testing.assert_array_equal(x, y)
    a0 = c["emu"].track(c["q0"], c["ft"], held[0], None, **c["kw"], **CONV, lengths=ln)
    b2 = c["emu"].track(c["q0"], c["ft"], np.repeat(held[:1], T, axis=0), None, **c["kw"], **CONV, lengths=ln, posture_form=2)
    for x, y in zip(a0, b2):
        np.testing.assert_array_equal(x, y)


def _two_posture_case(dtype, B=48, T=5, seed=3):
    """A 7-hinge chain with a PostureTask and a DampingTask (P = 2: slot 0 the posture target, slot 1 the damping task's qpos0)."""
    import mink_b200 as mink
    from mink_b200._abi import spec_from_workload
    from mink_b200.workloads import make_inputs
    from oracle.ikoracle import Oracle
    from tests.emu_posture_lib import PostureEmu
    from tests.helpers import chain_xml, task_frames

    fm = mink.flatten(mink.Model.from_xml_string(chain_xml(7, seed=seed)))
    wl = dict(robot="chain", key=None, frames=[dict(name="tip", type="site", position_cost=1.0, orientation_cost=1.0, lm_damping=1.0)],
              posture=dict(cost=5e-2), damping_task=dict(cost=0.3), com=None, limits=[dict(kind="configuration", gain=0.95)],
              dt=2e-2, damping=1e-3)
    spec = spec_from_workload(fm, wl)
    assert spec.nposture == 2
    orc = Oracle(fm.to_blob(), spec, fm.nq, fm.nv)
    frames = task_frames(wl, fm)
    inp = make_inputs(fm, wl, B, lambda qq: orc.fk(qq, frames), seed=seed, sigma=0.3)
    rng = np.random.default_rng(seed)
    path = inp["q"][:, None, :] + np.cumsum(rng.normal(0.0, 0.08, size=(B, T, fm.nq)), axis=1)
    poses, _ = orc.fk(path.reshape(B * T, fm.nq), frames)
    ft = np.asarray(poses, dtype).reshape(B, T, -1, 7)
    emu = PostureEmu(fm.to_blob(), spec, fm.nq, fm.nv)
    return dict(emu=emu, fm=fm, q0=inp["q"].astype(dtype), ft=ft, path=path.astype(dtype), kw=dict(dt=wl["dt"], damping=wl["damping"]),
                B=B, T=T, ct=None)


@pytest.mark.parametrize("dtype", [np.float32, np.float64], ids=["f32", "f64"])
def test_two_posture_tasks(dtype):
    """One held target (the DampingTask's qpos0) next to a sequence (the PostureTask follows the joint path): the sequence's rows
    must land in slot 0 of every frame and the held rows in slot 1."""
    c = _two_posture_case(dtype)
    B, T, nq = c["B"], c["T"], c["fm"].nq
    qpos0 = np.broadcast_to(np.asarray(c["fm"].qpos0, dtype), (B, T, nq))
    seq = np.stack([c["path"], qpos0], axis=2)                    # [B, T, 2, nq]
    ln = np.full(B, T, np.int32)
    ln[:3] = [0, T, 1]
    c["ft"] = np.ascontiguousarray(c["ft"])
    loop = _per_frame(c, lambda t: seq[:, t])
    out = c["emu"].track(c["q0"], c["ft"], seq, None, **c["kw"], **CONV, lengths=ln, posture_form=3)
    _check_equal(c, loop, out, ln)
    swapped = c["emu"].track(c["q0"], c["ft"], seq[:, :, ::-1], None, **c["kw"], **CONV, lengths=ln, posture_form=3)
    assert not np.array_equal(swapped[1][ln > 1], out[1][ln > 1])


def test_sequence_against_oracle():
    """The C oracle's fp64 converge loop frame by frame, each frame with its posture target: iteration counts agree on
    >= 99.5 % of (b, t); where an instance's counts agree up to frame t, q_traj[b][t] is within 1e-3 (the bar of
    test_emulated_track_against_oracle)."""
    c = _case("ur5e", np.float32, B=200 + 3, T=8, seed=44)
    _, q_traj, it, _, _ = c["emu"].track(c["q0"], c["ft"], c["pseq"], None, **c["kw"], **CONV, posture_form=3)
    q = c["q0"].astype(np.float64)
    q_ref, it_ref = np.zeros(q_traj.shape), np.zeros_like(it)
    for t in range(c["T"]):
        q, it_ref[:, t], _, _ = c["orc"].converge(q, c["ft"][:, t].astype(np.float64), c["pseq"][:, t].astype(np.float64), None,
                                                  **c["kw"], **CONV)
        q_ref[:, t] = q
    same = it == it_ref
    assert same.mean() >= 0.995, f"{int((~same).sum())} of {same.size} iteration counts differ"
    upto = np.cumprod(same, axis=1).astype(bool)
    np.testing.assert_allclose(q_traj[upto], q_ref[upto], atol=1e-3)
