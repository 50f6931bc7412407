"""Per-instance posture weights (bik_converge_weighted_ex / bik_track_weighted_ex) through the pass loops compiled for the host
(tests/host_emu/emu_posture_weights.cpp), no GPU needed.

Instance b solves the QP whose PostureTask / DampingTask cost on dof d is cost[p][d] * w[b][p][d]: all-ones weights give the
unweighted loops bit for bit, random weights give what the fp64 oracle gives with those costs, a weight of 0 on a DampingTask
gives the problem without it, out-of-range weights are clamped and flagged, and bik_track with per-frame weights is one converge
per frame.  Cases: ur5e_damp (a DampingTask alone), TidyBot with the examples' immobile-base DampingTask, G1 with a
Levenberg-Marquardt term on its posture (all three on the small-group K2), and Spot with a PostureTask (with a
Levenberg-Marquardt term) and a DampingTask added (collision rows: the general K2).
"""

import copy

import numpy as np
import pytest

from mink_b200._abi import TASK_POSTURE
from mink_b200.workloads import WORKLOADS
from tests.emu_posture_weights_lib import PATH_GENERAL, PostureWeightedEmu

CONV = dict(max_iters=10, pos_threshold=2e-3, ori_threshold=2e-3)
BAD_WEIGHT = 32
NAMES = ["ur5e_damp", "tidybot", "g1", "spot"]


def _workload(name):
    wl = WORKLOADS[name]
    if name == "tidybot":   # examples/mobile_tidybot.py: DampingTask(model, immobile_base_cost), cost 100 on the base's three dofs
        return dict(wl, damping_task=dict(cost=[100.0] * 3 + [0.0] * 15))
    if name == "g1":
        return dict(wl, posture=dict(wl["posture"], lm_damping=0.5))
    if name == "spot":
        return dict(wl, posture=dict(cost=1e-2, lm_damping=1.0), damping_task=dict(cost=0.1))
    return wl


def _posture_slots(spec):
    """Indices into spec.tasks of the posture-type tasks, in the order of posture_targets / posture_weights."""
    return [i for i, t in enumerate(spec.tasks) if t.kind == TASK_POSTURE]


def _case(name, dtype, B, T, seed, wl=None):
    """Targets from the oracle's FK along a seeded joint path (as tests.helpers.track_case); pt [B, P, nq]: each instance's q0
    for a PostureTask, qpos0 for a DampingTask (gain 0); pseq [B, T, P, nq]: the PostureTask's target drifting away from q0."""
    from mink_b200._abi import spec_from_workload
    from mink_b200.workloads import load_flat, make_inputs, task_frames
    from oracle.ikoracle import Oracle

    wl = wl or _workload(name)
    fm = load_flat(wl["robot"])
    spec = spec_from_workload(fm, wl)
    orc = Oracle(fm.to_blob(), spec, fm.nq, fm.nv)
    frames = task_frames(wl, fm)
    inp = make_inputs(fm, wl, B, lambda qq: orc.fk(qq, frames), seed=seed, sigma=0.3)
    rng = np.random.default_rng(seed + 1)
    path = np.repeat(inp["q"][:, None, :], T, axis=1)
    frac = np.arange(1, T + 1) / T
    slots = _posture_slots(spec)
    damping = [spec.tasks[i].gain == 0.0 for i in slots]
    pt = np.stack([np.broadcast_to(fm.qpos0, inp["q"].shape) if d else inp["q"] for d in damping], axis=1).astype(dtype) if slots else None
    pseq = np.repeat(pt[:, None], T, axis=1).astype(np.float64) if slots else None
    for n in range(fm.nnode):
        if int(fm.node_type[n]) >= 2:   # hinge / slide
            a = int(fm.node_qadr[n])
            path[:, :, a] += rng.normal(0.0, 0.3, size=B)[:, None] * frac[None, :]
            for p, d in enumerate(damping):
                if not d:
                    pseq[:, :, p, a] += np.cumsum(rng.normal(0.0, 0.05, size=(B, T)), axis=1)
    poses, com = orc.fk(path.reshape(B * T, fm.nq), frames)
    ft = np.asarray(poses, dtype).reshape(B, T, -1, 7)
    ct = np.asarray(com, dtype).reshape(B, T, -1, 3) if spec.ncom else None
    return dict(wl=wl, fm=fm, spec=spec, orc=orc, emu=PostureWeightedEmu(fm.to_blob(), spec, fm.nq, fm.nv), q0=inp["q"].astype(dtype),
                ft=ft, ct=ct, pt=pt, pseq=None if pseq is None else pseq.astype(dtype), damping=damping,
                kw=dict(dt=wl["dt"], damping=wl["damping"]), B=B, T=T, P=len(slots), nv=fm.nv)


def _at(a, t):
    return None if a is None else a[:, t]


def _eq(a, b):
    np.testing.assert_array_equal(a, b)


def _lengths(B, T, seed):
    ln = np.random.default_rng(seed).integers(0, T + 1, size=B).astype(np.int32)
    ln[:3] = [0, T, 1]
    return ln


@pytest.mark.parametrize("name", NAMES)
def test_precision_choice_unchanged(name):
    """With posture weights K1's precision for fp32 callers assumes every posture weight may be 0 (reg = damping); on these
    cases that choice is the one made without them (G1: 200^2 / 0.1 = 4e5 < 1e6; Spot: fp64 for its collision rows)."""
    c = _case(name, np.float32, B=4, T=1, seed=1)
    without, with_pw = c["emu"].k1_double(c["kw"]["damping"])
    assert without == with_pw
    assert with_pw == (name == "spot")


@pytest.mark.parametrize("dtype", [np.float32, np.float64], ids=["f32", "f64"])
@pytest.mark.parametrize("name", NAMES)
def test_ones_are_the_identity(name, dtype):
    """All-ones posture weights give the ..._weighted loops bit for bit (random task weights alongside), for converge and for
    track with ragged lengths; on the small-group cases also with K2 forced onto the general path."""
    from tests.emu_weights_lib import WeightedEmu

    c = _case(name, dtype, B=40 + 3, T=4, seed=3)
    B, T, P, nv, K = c["B"], c["T"], c["P"], c["nv"], c["spec"].nrows
    w = np.random.default_rng(4).uniform(0.2, 1.0, size=(B, T, K)).astype(dtype)
    wemu = WeightedEmu(c["fm"].to_blob(), c["spec"], c["fm"].nq, nv)
    ref = wemu.converge(c["q0"], c["ft"][:, 0], c["pt"], _at(c["ct"], 0), w[:, 0], **c["kw"], **CONV)
    got = c["emu"].converge(c["q0"], c["ft"][:, 0], c["pt"], _at(c["ct"], 0), np.ones((B, P, nv), dtype), **c["kw"], **CONV, weights=w[:, 0])
    for x, y in zip(got, ref):
        _eq(x, y)
    ln = _lengths(B, T, 5)
    ref = wemu.track(c["q0"], c["ft"], c["pt"], c["ct"], w, **c["kw"], **CONV, lengths=ln)
    got = c["emu"].track(c["q0"], c["ft"], c["pt"], c["ct"], np.ones((B, T, P, nv), dtype), **c["kw"], **CONV, lengths=ln, weights=w)
    for x, y in zip(got, ref):
        _eq(x, y)
    if name != "spot":
        ref = c["emu"].converge(c["q0"], c["ft"][:, 0], c["pt"], None, None, **c["kw"], **CONV, weights=w[:, 0], path=PATH_GENERAL)
        got = c["emu"].converge(c["q0"], c["ft"][:, 0], c["pt"], None, np.ones((B, P, nv), dtype), **c["kw"], **CONV, weights=w[:, 0],
                                path=PATH_GENERAL)
        for x, y in zip(got, ref):
            _eq(x, y)


def _scaled_spec(spec, om):
    """The problem with the dof costs of posture-type task p multiplied by om[p] [nv]."""
    s = copy.deepcopy(spec)
    for p, i in enumerate(_posture_slots(spec)):
        s.tasks[i].dof_cost = np.asarray(spec.tasks[i].dof_cost, np.float64) * om[p]
    return s


@pytest.mark.parametrize("dtype", [np.float64, np.float32], ids=["f64", "f32"])
@pytest.mark.parametrize("name", NAMES)
def test_weights_are_costs(name, dtype):
    """One step of instance b with posture weights w[b] in [0.1, 1] is the fp64 oracle's step with the costs cost * w[b]:
    1e-8 rad in fp64 (plus 2e-9 relative: on ur5e_damp, where |q| reaches 5 rad, the unweighted loop itself is 1.0e-8 rad
    off the oracle), 1e-4 rad in fp32.  In fp64 the whole loop also takes the oracle's iteration counts."""
    from oracle.ikoracle import Oracle

    c = _case(name, dtype, B=6, T=1, seed=21)
    B, P, nv = c["B"], c["P"], c["nv"]
    om = np.random.default_rng(5).uniform(0.1, 1.0, size=(B, P, nv)).astype(dtype)
    ft, ct = c["ft"][:, 0], _at(c["ct"], 0)
    q1, _, st = c["emu"].converge(c["q0"], ft, c["pt"], ct, om, **c["kw"], max_iters=1, pos_threshold=0.0, ori_threshold=0.0)
    assert not (st & ~16).any(), st
    qn, itn, _ = c["emu"].converge(c["q0"], ft, c["pt"], ct, om, **c["kw"], **CONV)
    f64 = lambda a: None if a is None else np.asarray(a, np.float64)
    tol = 1e-8 if dtype == np.float64 else 1e-4
    for b in range(B):
        orc = Oracle(c["fm"].to_blob(), _scaled_spec(c["spec"], om[b].astype(np.float64)), c["fm"].nq, nv)
        args = (f64(c["q0"][b:b + 1]), f64(ft[b:b + 1]), f64(c["pt"][b:b + 1]), None if ct is None else f64(ct[b:b + 1]))
        _, q_ref, st_ref, _ = orc.step(*args, **c["kw"], nsteps=1, integrate=True)
        assert not st_ref.any()
        np.testing.assert_allclose(q1[b], q_ref[0], atol=tol, rtol=2e-9 if dtype == np.float64 else 0)
        if dtype == np.float64:
            _, it_ref, _, _ = orc.converge(*args, **c["kw"], **CONV)
            assert itn[b] == it_ref[0], (b, itn[b], it_ref[0])


def _without_damping(c):
    """The case's problem without its DampingTask, and the posture targets / slots that go with it."""
    wl = dict(c["wl"], damping_task=None)
    keep = [p for p, d in enumerate(c["damping"]) if not d]
    return _case_problem(c, wl), keep


def _case_problem(c, wl):
    from mink_b200._abi import spec_from_workload

    spec = spec_from_workload(c["fm"], wl)
    return PostureWeightedEmu(c["fm"].to_blob(), spec, c["fm"].nq, c["nv"])


@pytest.mark.parametrize("dtype", [np.float64, np.float32], ids=["f64", "f32"])
@pytest.mark.parametrize("name", ["ur5e_damp", "tidybot", "spot"])
def test_zero_weight_drops_the_damping_task(name, dtype):
    """The fixed-base batch: DampingTask weight 1 on even instances, 0 on odd ones (PostureTask weight 1).  Even instances give
    the problem with the task bit for bit; odd ones the problem without it, 1e-9 rad in fp64 and 1e-5 in fp32, with the same
    iteration counts and status; converge and track."""
    c = _case(name, dtype, B=24, T=3, seed=8)
    B, T, P, nv = c["B"], c["T"], c["P"], c["nv"]
    d = c["damping"].index(True)
    om = np.ones((B, T, P, nv), dtype)
    om[1::2, :, d] = 0.0
    small, keep = _without_damping(c)
    pt_small = c["pt"][:, keep] if keep else None
    tol = 1e-9 if dtype == np.float64 else 1e-5
    odd, even = np.arange(B) % 2 == 1, np.arange(B) % 2 == 0

    q, it, st = c["emu"].converge(c["q0"], c["ft"][:, 0], c["pt"], _at(c["ct"], 0), om[:, 0], **c["kw"], **CONV)
    q_f, it_f, st_f = c["emu"].converge(c["q0"], c["ft"][:, 0], c["pt"], _at(c["ct"], 0), None, **c["kw"], **CONV)
    q_s, it_s, st_s = small.converge(c["q0"], c["ft"][:, 0], pt_small, _at(c["ct"], 0), None, **c["kw"], **CONV)
    _eq(q[even], q_f[even]); _eq(it[even], it_f[even]); _eq(st[even], st_f[even])
    np.testing.assert_allclose(q[odd], q_s[odd], atol=tol, rtol=0)
    _eq(it[odd], it_s[odd]); _eq(st[odd], st_s[odd])
    assert not np.allclose(q_f[odd], q_s[odd], atol=100 * tol, rtol=0)   # the task does change the result

    _, q_traj, it, st, _ = c["emu"].track(c["q0"], c["ft"], c["pt"], c["ct"], om, **c["kw"], **CONV)
    _, q_traj_s, it_s, st_s, _ = small.track(c["q0"], c["ft"], pt_small, c["ct"], None, **c["kw"], **CONV)
    np.testing.assert_allclose(q_traj[odd], q_traj_s[odd], atol=10 * tol, rtol=0)
    _eq(it[odd], it_s[odd]); _eq(st[odd], st_s[odd])


@pytest.mark.parametrize("dtype", [np.float32, np.float64], ids=["f32", "f64"])
@pytest.mark.parametrize("name", ["g1", "spot"])
def test_out_of_range_and_nan_weights_are_clamped_and_flagged(name, dtype):
    """Posture weights above 1, below 0 or NaN run as 1, 0 and 0, and only their instances (in track mode: their frames) get
    BIK_STATUS_BAD_WEIGHT; g1 on the small-group K2, spot on the general one."""
    c = _case(name, dtype, B=12, T=2, seed=9)
    B, T, P, nv = c["B"], c["T"], c["P"], c["nv"]
    rng = np.random.default_rng(10)
    om = rng.uniform(0.2, 1.0, size=(B, T, P, nv)).astype(dtype)
    bad, clamped = om.copy(), om.copy()
    bad[1, :, 0, 6], clamped[1, :, 0, 6] = 1.5, 1.0
    bad[4, :, P - 1, 7], clamped[4, :, P - 1, 7] = -0.25, 0.0
    bad[7, :, 0, nv - 1], clamped[7, :, 0, nv - 1] = np.nan, 0.0
    bad[9, 1, 0, 8], clamped[9, 1, 0, 8] = np.inf, 1.0      # only frame 1 of instance 9
    flagged = np.zeros(B, bool)
    flagged[[1, 4, 7]] = True
    ct0 = _at(c["ct"], 0)
    q, it, st = c["emu"].converge(c["q0"], c["ft"][:, 0], c["pt"], ct0, bad[:, 0], **c["kw"], **CONV)
    q_c, it_c, st_c = c["emu"].converge(c["q0"], c["ft"][:, 0], c["pt"], ct0, clamped[:, 0], **c["kw"], **CONV)
    _eq(q, q_c)
    _eq(it, it_c)
    assert not (st_c & BAD_WEIGHT).any()
    _eq(st, st_c | np.where(flagged, BAD_WEIGHT, 0))
    _, q_traj, it, st, _ = c["emu"].track(c["q0"], c["ft"], c["pt"], c["ct"], bad, **c["kw"], **CONV)
    _, q_traj_c, it_c, st_c, _ = c["emu"].track(c["q0"], c["ft"], c["pt"], c["ct"], clamped, **c["kw"], **CONV)
    _eq(q_traj, q_traj_c)
    _eq(it, it_c)
    flagged_t = np.repeat(flagged[:, None], T, axis=1)
    flagged_t[9, 1] = True
    _eq(st, st_c | np.where(flagged_t, BAD_WEIGHT, 0))


@pytest.mark.parametrize("dtype", [np.float32, np.float64], ids=["f32", "f64"])
@pytest.mark.parametrize("name", ["tidybot", "g1", "spot"])
@pytest.mark.parametrize("seq", [False, True], ids=["held", "sequence"])
def test_track_equals_per_frame_converge(name, dtype, seq):
    """bik_track_weighted_ex with per-frame posture weights [B, T, P, nv] equals one converge per frame with frame t's weights,
    bit for bit, with ragged lengths; with `sequence` the posture targets follow a BIK_POSTURE_SEQ_BATCHED sequence too."""
    c = _case(name, dtype, B=32 + 5, T=4, seed=12)
    B, T, P, nv = c["B"], c["T"], c["P"], c["nv"]
    om = np.random.default_rng(13).uniform(0.0, 1.0, size=(B, T, P, nv)).astype(dtype)
    om[::3, :, :, :5] = 0.0
    ln = _lengths(B, T, 2)
    pts = (lambda t: c["pseq"][:, t]) if seq else (lambda t: c["pt"])
    q = c["q0"]
    q_loop, it_loop, st_loop = np.zeros((B, T, c["fm"].nq), q.dtype), np.zeros((B, T), np.int32), np.zeros((B, T), np.int32)
    for t in range(T):
        q, it_loop[:, t], st_loop[:, t] = c["emu"].converge(q, c["ft"][:, t], pts(t), _at(c["ct"], t), om[:, t], **c["kw"], **CONV)
        q_loop[:, t] = q
    q_end, q_traj, it, st, passes = c["emu"].track(c["q0"], c["ft"], c["pseq"] if seq else c["pt"], c["ct"], om, **c["kw"], **CONV,
                                                   lengths=ln, posture_form=3 if seq else None)
    has = np.arange(T)[None, :] < ln[:, None]
    _eq(q_traj[has], q_loop[has])
    _eq(it[has], it_loop[has])
    _eq(st[has], st_loop[has])
    assert np.isnan(q_traj[~has]).all() and (it[~has] == -1).all() and (st[~has] == -1).all()
    q_ref = np.where(ln[:, None] > 0, q_loop[np.arange(B), np.maximum(ln - 1, 0)], c["q0"])
    _eq(q_end, q_ref)
