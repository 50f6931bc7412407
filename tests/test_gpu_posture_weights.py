"""Per-instance posture weights on the device: bik_step_weighted_ex / bik_converge_weighted_ex / bik_track_weighted_ex (and
their fp64 forms) through Problem.step / converge / track, and the `posture_weights=` mapping of solve_ik / converge_ik /
track_ik.

The checks of tests/test_posture_weights_cpu.py, on the device and on the same cases: all-ones weights give the ..._weighted
entry points bit for bit (also with K2 forced onto the general path), weights are costs against the fp64 oracle, a weight of
0 on a DampingTask drops it, out-of-range weights are clamped and flagged, bik_track_weighted_ex is one converge per frame.
Then the cached converge graph following the posture-weights buffer, and the TidyBot fixed-base batch of the reference's
mobile examples through converge_ik.
"""

import os

import numpy as np
import pytest

torch = pytest.importorskip("torch")
pytestmark = pytest.mark.gpu

from tests.test_posture_weights_cpu import BAD_WEIGHT, NAMES, _case as _emu_case, _scaled_spec, _workload  # noqa: E402

CONV = dict(max_iters=10, pos_threshold=2e-3, ori_threshold=2e-3)
DT = {np.float32: torch.float32, np.float64: torch.float64}


def _problem(fm, spec, env=None):
    """A device Problem; env: variables set while it is created (BIK_K2_PATH is read then)."""
    from mink_b200.engine import DeviceModel, Problem

    old = {k: os.environ.get(k) for k in (env or {})}
    os.environ.update(env or {})
    try:
        return Problem(DeviceModel(fm, device=0), spec)
    finally:
        for k, v in old.items():
            if v is None:
                os.environ.pop(k, None)
            else:
                os.environ[k] = v


def _case(name, dtype, B, T, seed, env=None, wl=None):
    if not torch.cuda.is_available():
        pytest.skip("no CUDA device")
    c = _emu_case(name, dtype, B=B, T=T, seed=seed, wl=wl)
    c["prob"] = _problem(c["fm"], c["spec"], env)
    dev = lambda a: None if a is None else torch.tensor(np.ascontiguousarray(a), dtype=DT[dtype], device="cuda:0")
    c["d"] = dict(ft=dev(c["ft"]), ct=dev(c["ct"]), pt=dev(c["pt"]), pseq=dev(c["pseq"]))
    c["dev"] = dev
    return c


def _at(a, t):
    return None if a is None else a[:, t]


def _converge(c, pw=None, t=0, q=None, w=None, pt=None, prob=None, **kw):
    d = c["d"]
    q = c["dev"](c["q0"]) if q is None else q
    it, st = (prob or c["prob"]).converge(q, d["ft"][:, t], d["pt"] if pt is None else pt, _at(d["ct"], t), weights=w, posture_weights=pw,
                                          **c["kw"], **(kw or CONV))
    return q, it, st


def _equal(a, b):
    torch.testing.assert_close(a, b, rtol=0, atol=0, equal_nan=True)


@pytest.mark.parametrize("dtype", [np.float32, np.float64], ids=["f32", "f64"])
@pytest.mark.parametrize("name", NAMES)
def test_ones_are_the_identity(name, dtype):
    """All-ones posture weights: bit for bit the ..._weighted entry points (step, converge, track with ragged lengths)."""
    c = _case(name, dtype, B=200 + 3, T=4, seed=3)
    B, T, P, nv, K = c["B"], c["T"], c["P"], c["nv"], c["spec"].nrows
    w = c["dev"](np.random.default_rng(4).uniform(0.2, 1.0, size=(B, T, K)))
    ones = torch.ones((B, T, P, nv), dtype=DT[dtype], device="cuda:0")
    for x, y in zip(_converge(c, ones[:, 0].contiguous(), w=w[:, 0].contiguous()), _converge(c, w=w[:, 0].contiguous())):
        _equal(x, y)
    d = c["d"]
    q0, q1 = c["dev"](c["q0"]), c["dev"](c["q0"])
    r0 = c["prob"].step(q0, d["ft"][:, 0], d["pt"], _at(d["ct"], 0), **c["kw"], nsteps=3, integrate=True, posture_weights=ones[:, 0])
    r1 = c["prob"].step(q1, d["ft"][:, 0], d["pt"], _at(d["ct"], 0), **c["kw"], nsteps=3, integrate=True)
    for x, y in zip((q0,) + r0, (q1,) + r1):
        _equal(x, y)
    ln = torch.tensor(np.random.default_rng(5).integers(0, T + 1, size=B), dtype=torch.int32, device="cuda:0")
    q0, q1 = c["dev"](c["q0"]), c["dev"](c["q0"])
    r0 = c["prob"].track(q0, d["ft"], d["pt"], d["ct"], lengths=ln, weights=w, posture_weights=ones, **c["kw"], **CONV)
    r1 = c["prob"].track(q1, d["ft"], d["pt"], d["ct"], lengths=ln, weights=w, **c["kw"], **CONV)
    for x, y in zip((q0,) + r0[:3], (q1,) + r1[:3]):
        _equal(x, y)
    assert int(r0[3]) == int(r1[3])


@pytest.mark.parametrize("dtype", [np.float32, np.float64], ids=["f32", "f64"])
@pytest.mark.parametrize("name", ["ur5e_damp", "tidybot", "g1"])
def test_ones_are_the_identity_on_the_general_path(name, dtype):
    """The same with BIK_K2_PATH=dense, so that the general K2's posture-weighted instantiation runs these problems."""
    c = _case(name, dtype, B=100 + 3, T=1, seed=6, env={"BIK_K2_PATH": "dense"})
    ones = torch.ones((c["B"], c["P"], c["nv"]), dtype=DT[dtype], device="cuda:0")
    for x, y in zip(_converge(c, ones), _converge(c)):
        _equal(x, y)


@pytest.mark.parametrize("dtype", [np.float64, np.float32], ids=["f64", "f32"])
@pytest.mark.parametrize("name", NAMES)
def test_weights_are_costs(name, dtype):
    """bik_step_weighted_ex's dq and one converge step against the fp64 oracle with the costs cost * w[b]: 1e-8 rad (plus
    2e-9 relative, as on the host) in fp64, 1e-4 rad in fp32."""
    from oracle.ikoracle import Oracle

    c = _case(name, dtype, B=8, T=1, seed=21)
    fm, spec, B, P, nv = c["fm"], c["spec"], c["B"], c["P"], c["nv"]
    om = np.random.default_rng(5).uniform(0.1, 1.0, size=(B, P, nv)).astype(dtype)
    pw = c["dev"](om)
    d = c["d"]
    dq, st = c["prob"].step(c["dev"](c["q0"]), d["ft"][:, 0], d["pt"], _at(d["ct"], 0), **c["kw"], posture_weights=pw)
    q1, _, st1 = _converge(c, pw, max_iters=1, pos_threshold=0.0, ori_threshold=0.0)
    assert not st.any() and not (st1 & ~16).any()
    dq, q1 = dq.cpu().numpy(), q1.cpu().numpy()
    f64 = lambda a: None if a is None else np.asarray(a, np.float64)
    tol, rtol = (1e-8, 2e-9) if dtype == np.float64 else (1e-4, 0)
    for b in range(B):
        orc = Oracle(fm.to_blob(), _scaled_spec(spec, om[b].astype(np.float64)), fm.nq, nv)
        ct = None if c["ct"] is None else f64(c["ct"][b:b + 1, 0])
        dq_ref, q_ref, st_ref, _ = orc.step(f64(c["q0"][b:b + 1]), f64(c["ft"][b:b + 1, 0]), f64(c["pt"][b:b + 1]), ct, **c["kw"],
                                            nsteps=1, integrate=True)
        assert not st_ref.any()
        np.testing.assert_allclose(dq[b], dq_ref[0], atol=tol, rtol=0)
        np.testing.assert_allclose(q1[b], q_ref[0], atol=tol, rtol=rtol)


@pytest.mark.parametrize("dtype", [np.float64, np.float32], ids=["f64", "f32"])
@pytest.mark.parametrize("name", ["ur5e_damp", "tidybot", "spot"])
def test_zero_weight_drops_the_damping_task(name, dtype):
    """DampingTask weight 1 on even instances, 0 on odd ones: even instances give the problem with the task bit for bit, odd
    ones the problem without it (1e-9 rad in fp64, 1e-5 in fp32), with the same iteration counts and status."""
    c = _case(name, dtype, B=256, T=1, seed=8)
    B, P, nv = c["B"], c["P"], c["nv"]
    dmp = c["damping"].index(True)
    pw = torch.ones((B, P, nv), dtype=DT[dtype], device="cuda:0")
    pw[1::2, dmp] = 0.0
    from mink_b200._abi import spec_from_workload

    keep = [p for p, dd in enumerate(c["damping"]) if not dd]
    small = _problem(c["fm"], spec_from_workload(c["fm"], dict(c["wl"], damping_task=None)))
    q, it, st = _converge(c, pw)
    q_f, it_f, st_f = _converge(c)
    q_s, it_s, st_s = _converge(c, prob=small, pt=c["d"]["pt"][:, keep].contiguous() if keep else None)
    _equal(q[0::2], q_f[0::2]); _equal(it[0::2], it_f[0::2]); _equal(st[0::2], st_f[0::2])
    tol = 1e-9 if dtype == np.float64 else 1e-5
    assert (q[1::2] - q_s[1::2]).abs().max().item() <= tol
    _equal(it[1::2], it_s[1::2]); _equal(st[1::2], st_s[1::2])
    assert (q_f[1::2] - q_s[1::2]).abs().max().item() > 100 * tol


@pytest.mark.parametrize("dtype", [np.float32, np.float64], ids=["f32", "f64"])
@pytest.mark.parametrize("name", ["g1", "spot"])
def test_out_of_range_and_nan_weights_are_clamped_and_flagged(name, dtype):
    c = _case(name, dtype, B=64, T=2, seed=9)
    B, T, P, nv = c["B"], c["T"], c["P"], c["nv"]
    om = np.random.default_rng(10).uniform(0.2, 1.0, size=(B, T, P, nv)).astype(dtype)
    bad, clamped = om.copy(), om.copy()
    bad[1, :, 0, 6], clamped[1, :, 0, 6] = 1.5, 1.0
    bad[4, :, P - 1, 7], clamped[4, :, P - 1, 7] = -0.25, 0.0
    bad[7, :, 0, nv - 1], clamped[7, :, 0, nv - 1] = np.nan, 0.0
    bad[9, 1, 0, 8], clamped[9, 1, 0, 8] = np.inf, 1.0      # only frame 1 of instance 9
    flagged = np.zeros(B, np.int32)
    flagged[[1, 4, 7]] = BAD_WEIGHT
    q, it, st = _converge(c, c["dev"](bad[:, 0]))
    q_c, it_c, st_c = _converge(c, c["dev"](clamped[:, 0]))
    _equal(q, q_c)
    _equal(it, it_c)
    assert not (st_c & BAD_WEIGHT).any()
    np.testing.assert_array_equal(st.cpu().numpy(), st_c.cpu().numpy() | flagged)
    d = c["d"]
    _, st = c["prob"].step(c["dev"](c["q0"]), d["ft"][:, 0], d["pt"], _at(d["ct"], 0), **c["kw"], posture_weights=c["dev"](bad[:, 0]))
    assert ((st.cpu().numpy() & BAD_WEIGHT) == flagged).all()
    r = c["prob"].track(c["dev"](c["q0"]), d["ft"], d["pt"], d["ct"], posture_weights=c["dev"](bad), **c["kw"], **CONV)
    r_c = c["prob"].track(c["dev"](c["q0"]), d["ft"], d["pt"], d["ct"], posture_weights=c["dev"](clamped), **c["kw"], **CONV)
    _equal(r[0], r_c[0])
    flagged_t = np.repeat(flagged[:, None], T, axis=1)
    flagged_t[9, 1] = BAD_WEIGHT
    np.testing.assert_array_equal(r[2].cpu().numpy(), r_c[2].cpu().numpy() | flagged_t)


@pytest.mark.parametrize("dtype", [np.float32, np.float64], ids=["f32", "f64"])
@pytest.mark.parametrize("name", ["tidybot", "g1", "spot"])
@pytest.mark.parametrize("seq", [False, True], ids=["held", "sequence"])
def test_track_equals_per_frame_converge(name, dtype, seq):
    """bik_track_weighted_ex with [B, T, P, nv] weights is bit for bit one converge per frame with frame t's weights, with
    ragged lengths; with `sequence` the posture targets follow a BIK_POSTURE_SEQ_BATCHED sequence too."""
    c = _case(name, dtype, B=300 + 5, T=4, seed=12)
    B, T, P, nv = c["B"], c["T"], c["P"], c["nv"]
    om = np.random.default_rng(13).uniform(0.0, 1.0, size=(B, T, P, nv)).astype(dtype)
    om[::3, :, :, :5] = 0.0
    pw = c["dev"](om)
    ln = np.random.default_rng(2).integers(0, T + 1, size=B).astype(np.int32)
    d = c["d"]
    q = c["dev"](c["q0"])
    q_loop = torch.zeros((B, T, c["fm"].nq), dtype=q.dtype, device="cuda:0")
    it_loop = torch.zeros((B, T), dtype=torch.int32, device="cuda:0")
    st_loop = torch.zeros((B, T), dtype=torch.int32, device="cuda:0")
    for t in range(T):
        pt = d["pseq"][:, t].contiguous() if seq else None
        _, it_loop[:, t], st_loop[:, t] = _converge(c, pw[:, t].contiguous(), t=t, q=q, pt=pt)
        q_loop[:, t] = q
    q_end = c["dev"](c["q0"])
    q_traj, it, st, _ = c["prob"].track(q_end, d["ft"], d["pseq"] if seq else d["pt"], d["ct"], lengths=torch.tensor(ln, device="cuda:0"),
                                        posture_weights=pw, posture_seq=seq, **c["kw"], **CONV)
    has = torch.tensor(np.arange(T)[None, :] < ln[:, None], device="cuda:0")
    _equal(q_traj[has], q_loop[has])
    _equal(it[has], it_loop[has])
    _equal(st[has], st_loop[has])


def test_cached_graph_follows_the_posture_weights_buffer():
    """Converge calls on one problem alternating between two posture-weights buffers, then the unweighted call, give what a
    problem without a cached graph gives; so does rewriting a buffer in place between two calls."""
    c = _case("g1", np.float32, B=256 + 7, T=1, seed=30)
    B, P, nv = c["B"], c["P"], c["nv"]
    rng = np.random.default_rng(31)
    pa, pb = (c["dev"](rng.uniform(0.0, 1.0, size=(B, P, nv))) for _ in range(2))
    fresh = lambda pw: _converge(c, pw, prob=_problem(c["fm"], c["spec"]))
    ref_a, ref_b, ref_0 = fresh(pa), fresh(pb), fresh(None)
    for pw, ref in ((pa, ref_a), (pb, ref_b), (pa, ref_a), (None, ref_0), (pb, ref_b)):
        for x, y in zip(_converge(c, pw), ref):
            _equal(x, y)
    pb.copy_(pa)
    for x, y in zip(_converge(c, pb), ref_a):
        _equal(x, y)


def test_c_abi_rejects_posture_weights_without_posture_tasks():
    """A non-null posture-weights buffer on a problem without PostureTask / DampingTask: BIK_ERR_INVALID, nothing runs."""
    import ctypes as C

    from mink_b200 import _lib

    c = _case("spot", np.float32, B=4, T=1, seed=1, wl=dict(_workload("spot"), posture=None, damping_task=None))
    assert c["P"] == 0
    prob, d = c["prob"], c["d"]
    q = c["dev"](c["q0"])
    inp, keep, _, _ = prob._inputs(None, d["ft"][:, 0], None, _at(d["ct"], 0), dtype=q.dtype)
    junk = torch.ones(64, dtype=torch.float32, device="cuda:0")
    it = torch.zeros(4, dtype=torch.int32, device="cuda:0")
    st = torch.zeros(4, dtype=torch.int32, device="cuda:0")
    rc = prob.lib.bik_converge_weighted_ex(prob.handle, 4, q.data_ptr(), C.byref(inp), None, junk.data_ptr(), float(c["kw"]["dt"]),
                                           float(c["kw"]["damping"]), 10, 2e-3, 2e-3, 1, it.data_ptr(), st.data_ptr(), None)
    assert rc == -1 and b"posture" in _lib.load().bik_last_error()
    with pytest.raises(ValueError):
        prob.converge(q, d["ft"][:, 0], None, _at(d["ct"], 0), posture_weights=junk, **c["kw"])


def _tidybot_api(fm, q, target, base_fixed_cost=100.0):
    """The reference's mobile TidyBot example (examples/mobile_tidybot.py): pinch-site FrameTask, PostureTask, and a DampingTask
    with cost 100 on the base's three dofs that holds the base still."""
    import mink_b200 as mink
    from mink_b200.lie import SE3

    cfg = mink.Configuration(fm, q)
    ee = mink.FrameTask("pinch_site", "site", position_cost=1.0, orientation_cost=1.0, lm_damping=1.0)
    ee.set_target(SE3(wxyz_xyz=target))
    post = mink.PostureTask(fm, cost=np.array([0.0] * 3 + [1e-3] * 15))
    post.set_target(np.asarray(fm.key("home"), np.float64))
    cost = np.zeros(fm.nv)
    cost[:3] = base_fixed_cost
    damp = mink.DampingTask(fm, cost)
    return mink, cfg, ee, post, damp, [mink.ConfigurationLimit(fm, gain=0.95)]


def test_tidybot_fixed_base_batch():
    """One problem with [FrameTask, PostureTask, DampingTask(immobile_base_cost)], damping weight 1 on even instances and 0 on
    odd ones: each instance's converge_ik equals the separate problem with (even) or without (odd) the DampingTask, 1e-9 rad
    in fp64; the even instances' base barely moves next to the odd ones'."""
    from tests.helpers import load_case

    if not torch.cuda.is_available():
        pytest.skip("no CUDA device")
    wl, fm, spec, g = load_case("tidybot")
    dt, damping = float(wl["dt"]), float(wl["damping"])
    B = 16
    c = _emu_case("tidybot", np.float64, B=B, T=1, seed=40)
    q0 = torch.tensor(c["q0"], dtype=torch.float64, device="cuda:0")
    targets = c["ft"][:, 0, 0]
    mink, cfg, ee, post, damp, limits = _tidybot_api(fm, q0.clone(), targets)
    w = np.ones((B, fm.nv))
    w[1::2] = 0.0
    conv = dict(max_iters=20, pos_threshold=1e-4, ori_threshold=1e-4)
    it, ok = mink.converge_ik(cfg, [ee, post, damp], dt, damping=damping, limits=limits, posture_weights={damp: w}, **conv)
    q = cfg.q_device.cpu().numpy()
    base_move = np.abs(q[:, :3] - c["q0"][:, :3]).max(axis=1)
    for b in range(B):
        mink, cfg1, ee1, post1, damp1, limits1 = _tidybot_api(fm, c["q0"][b], targets[b])
        tasks1 = [ee1, post1, damp1] if b % 2 == 0 else [ee1, post1]
        it1, ok1 = mink.converge_ik(cfg1, tasks1, dt, damping=damping, limits=limits1, **conv)
        assert (int(it[b]), bool(ok[b])) == (it1, ok1), b
        np.testing.assert_allclose(q[b], cfg1.q, atol=1e-9, rtol=0)
    assert np.median(base_move[0::2]) < 0.1 * np.median(base_move[1::2]), base_move


def test_front_end_posture_weights():
    """solve_ik / converge_ik / track_ik with posture_weights={task: w}: a single (fp64) configuration equals the problem with
    the task's cost multiplied by w; batches take a float, [nv], [B, nv], and for track_ik [T, nv] and [B, T, nv]; wrong shapes
    and other task kinds are InvalidTarget; `weights=` still rejects a PostureTask; a bad weight fails the solve."""
    import mink_b200 as mink
    from mink_b200.exceptions import InvalidTarget
    from mink_b200.lie import SE3
    from tests.helpers import load_case

    if not torch.cuda.is_available():
        pytest.skip("no CUDA device")
    wl, fm, spec, g = load_case("ur5e")
    dt, damping = float(g["dt"]), float(g["damping"])
    nv = fm.nv

    def api(q, cost=1e-2):
        cfg = mink.Configuration(fm, q)
        ee = mink.FrameTask("attachment_site", "site", position_cost=1.0, orientation_cost=1.0, lm_damping=1.0)
        ee.set_target(SE3(wxyz_xyz=g["frame_targets"][0, 0]))
        post = mink.PostureTask(fm, cost=cost)
        post.set_target(g["posture_target"])
        return cfg, ee, post, [mink.ConfigurationLimit(fm, gain=0.95)]

    w = np.array([0.5, 0.25, 1.0, 0.75, 0.5, 0.125])   # exact in fp32
    for b in range(3):
        cfg, ee, post, limits = api(g["q"][b])
        v = mink.solve_ik(cfg, [ee, post], dt, damping=damping, limits=limits, posture_weights={post: w})
        cfg2, ee2, post2, limits2 = api(g["q"][b], cost=np.float32(1e-2) * w)
        v_ref = mink.solve_ik(cfg2, [ee2, post2], dt, damping=damping, limits=limits2)
        assert isinstance(v, np.ndarray) and v.dtype == np.float64
        np.testing.assert_allclose(v, v_ref, atol=1e-9, rtol=0)
        it, ok = mink.converge_ik(cfg, [ee, post], dt, damping=damping, limits=limits, posture_weights={post: w}, **CONV)
        it2, ok2 = mink.converge_ik(cfg2, [ee2, post2], dt, damping=damping, limits=limits2, **CONV)
        assert (it, ok) == (it2, ok2)
        np.testing.assert_allclose(cfg.q, cfg2.q, atol=1e-9, rtol=0)

    B, T = 4, 3
    qb = torch.tensor(g["q"][:B], dtype=torch.float32, device="cuda:0")
    wb = np.random.default_rng(1).uniform(0.2, 1.0, size=(B, nv))
    cfg, ee, post, limits = api(qb.clone())
    v = mink.solve_ik(cfg, [ee, post], dt, damping=damping, limits=limits, posture_weights={post: wb})
    for b in range(B):
        cfg1, ee1, post1, limits1 = api(qb[b:b + 1].clone())
        v1 = mink.solve_ik(cfg1, [ee1, post1], dt, damping=damping, limits=limits1, posture_weights={post1: wb[b]})
        _equal(v[b:b + 1], v1)
    for ws in (0.5, wb[0], wb):
        cfg, ee, post, limits = api(qb.clone())
        mink.converge_ik(cfg, [ee, post], dt, damping=damping, limits=limits, posture_weights={post: ws}, **CONV)
    seq = np.repeat(g["frame_targets"][0, 0][None], T, axis=0)
    wt = np.random.default_rng(2).uniform(0.2, 1.0, size=(B, T, nv))
    for ws in (0.5, wb[0], wb, wt[0], wt):
        cfg, ee, post, limits = api(qb.clone())
        q_traj, iters, ok = mink.track_ik(cfg, [ee, post], dt, {ee: seq}, damping=damping, limits=limits, posture_weights={post: ws}, **CONV)
        assert q_traj.shape == (B, T, fm.nq) and (iters >= 1).all()

    cfg, ee, post, limits = api(qb.clone())
    for bad in ({post: np.ones(nv + 1)}, {post: np.ones((B + 1, nv))}, {ee: np.ones(6)}):
        with pytest.raises(InvalidTarget):
            mink.solve_ik(cfg, [ee, post], dt, damping=damping, limits=limits, posture_weights=bad)
    with pytest.raises(InvalidTarget):
        mink.track_ik(cfg, [ee, post], dt, {ee: seq}, damping=damping, limits=limits, posture_weights={post: np.ones((T + 2, nv))})   # (T + 1 = B: a valid [B, nv])
    with pytest.raises(InvalidTarget):
        mink.solve_ik(cfg, [ee, post], dt, damping=damping, limits=limits, weights={post: np.ones(nv)})
    with pytest.raises(AssertionError):
        mink.solve_ik(cfg, [ee, post], dt, damping=damping, limits=limits, posture_weights={post: np.full(nv, np.nan)})
