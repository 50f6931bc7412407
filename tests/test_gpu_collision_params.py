"""Per-instance collision avoidance on the device: bik_step_coll / bik_converge_coll / bik_track_coll (and their fp64 forms)
through Problem.step / converge / track, and the `collision=` mapping of solve_ik / converge_ik / track_ik.

The checks of tests/test_collision_params_cpu.py, on the device and on the same cases: an all-ones mask with the problem's
distances gives the ..._bounded entry points bit for bit (also with K1 forced to fp32), random masks and distances give the
problems built with them bit for bit, non-finite distances are flagged, bik_track_coll is one collision converge per frame.
Then the cached converge graph following the collision buffers, the C ABI's refusals, a UR5e batch in which half of the
instances have no wall (converge_ik and track_ik), and the front end with CollisionAvoidanceLimit.pair_mask.
"""

import numpy as np
import pytest

torch = pytest.importorskip("torch")
pytestmark = pytest.mark.gpu

from tests.test_collision_params_cpu import (CONV, NAMES, NONFINITE, QP_MAXITER, _ccase, _random_distances,  # noqa: E402
                                             _random_masks, _rebuilt)
from tests.test_gpu_posture_weights import _problem  # noqa: E402
from tests.test_posture_weights_cpu import _lengths  # noqa: E402

DT = {np.float32: torch.float32, np.float64: torch.float64}
F32K1 = {"BIK_K1_PRECISION": "f32"}


def _case(name, dtype, B, T, seed, env=None):
    if not torch.cuda.is_available():
        pytest.skip("no CUDA device")
    c = _ccase(name, dtype, B=B, T=T, seed=seed)
    c["prob"] = _problem(c["fm"], c["spec"], env)
    dev = lambda a, dt=DT[dtype]: None if a is None else torch.tensor(np.ascontiguousarray(a), dtype=dt, device="cuda:0")
    c["d"] = dict(ft=dev(c["ft"]), ct=dev(c["ct"]), pt=dev(c["pt"]))
    c["dev"] = dev
    return c


def _at(a, t):
    return None if a is None else a[:, t]


def _dcoll(c, co):
    if co is None:
        return None
    en, dmin, ddet = co
    return (None if en is None else c["dev"](np.asarray(en, np.uint8), torch.uint8), c["dev"](dmin), c["dev"](ddet))


def _converge(c, co=None, prob=None, t=0, q=None, sl=slice(None), **kw):
    d = c["d"]
    q = c["dev"](c["q0"][sl]) if q is None else q
    pt = d["pt"] if d["pt"] is None else d["pt"][sl]
    ct = _at(d["ct"], t)
    it, st = (prob or c["prob"]).converge(q, d["ft"][sl, t], pt, None if ct is None else ct[sl], collision=co, **c["kw"], **(kw or CONV))
    return q, it, st


def _step(c, co=None, prob=None):
    d = c["d"]
    q = c["dev"](c["q0"])
    dq, st = (prob or c["prob"]).step(q, d["ft"][:, 0], d["pt"], _at(d["ct"], 0), nsteps=3, integrate=True, collision=co, **c["kw"])
    return q, dq, st


def _equal(a, b):
    torch.testing.assert_close(a, b, rtol=0, atol=0, equal_nan=True)


@pytest.mark.parametrize("dtype", [np.float32, np.float64], ids=["f32", "f64"])
@pytest.mark.parametrize("name", NAMES)
def test_all_ones_mask_is_the_bounded_entry_point(name, dtype):
    """An all-ones mask with the problem's own distances: bit for bit the entry points without collision arguments (step,
    converge, track with ragged lengths); fp32 callers also with K1 forced to fp32 (BIK_K1_PRECISION=f32)."""
    for env in ([None, F32K1] if dtype == np.float32 else [None]):
        c = _case(name, dtype, B=200 + 3, T=3, seed=3, env=env)
        B, T, lim, npairs = c["B"], c["T"], c["lim"], c["npairs"]
        dist = dtype == np.float64 or env is not None   # (an fp32 caller's fp64 K1 uses the problem's fp64 distances)
        co = _dcoll(c, (np.ones((B, npairs)), np.full(B, lim.minimum_distance) if dist else None,
                        np.full(B, lim.detection_distance) if dist else None))
        cot = _dcoll(c, (np.ones((B, T, npairs)), np.full((B, T), lim.minimum_distance) if dist else None,
                         np.full((B, T), lim.detection_distance) if dist else None))
        for x, y in zip(_step(c, co), _step(c)):
            _equal(x, y)
        for x, y in zip(_converge(c, co), _converge(c)):
            _equal(x, y)
        d = c["d"]
        ln = _lengths(B, T, 5)
        runs = [c["prob"].track(c["dev"](c["q0"]), d["ft"], d["pt"], d["ct"], lengths=ln, collision=x, **c["kw"], **CONV) for x in (cot, None)]
        for x, y in zip(*runs):
            _equal(x, y)


@pytest.mark.parametrize("dtype", [np.float32, np.float64], ids=["f32", "f64"])
@pytest.mark.parametrize("name", NAMES)
def test_random_masks_and_distances_are_the_rebuilt_problem(name, dtype):
    """Random masks (at least one pair), and random fp32-representable distances, give per instance what the problem built
    with those pairs and distances gives on the device, bit for bit, where neither run is flagged BIK_STATUS_QP_MAXITER."""
    c = _case(name, dtype, B=8, T=1, seed=21)
    B = c["B"]
    rng = np.random.default_rng(22)
    mask = _random_masks(rng, B, c["npairs"], 0.5)
    dmin, ddet = _random_distances(rng, c["lim"], B, dtype)
    for co in ((mask, None, None), (None, dmin, ddet), (mask, dmin, ddet)):
        q, it, st = _converge(c, _dcoll(c, co))
        compared = 0
        for b in range(B):
            _, spec_b = _rebuilt(c, None if co[0] is None else mask[b], None if co[1] is None else dmin[b], None if co[2] is None else ddet[b])
            qr, itr, str_ = _converge(c, None, prob=_problem(c["fm"], spec_b), sl=slice(b, b + 1))
            if int(st[b] | str_[0]) & QP_MAXITER:
                continue
            compared += 1
            _equal(q[b], qr[0]); _equal(it[b], itr[0]); _equal(st[b], str_[0])
        assert compared >= B // 2


@pytest.mark.parametrize("dtype", [np.float32, np.float64], ids=["f32", "f64"])
@pytest.mark.parametrize("name", NAMES)
def test_track_equals_per_frame_converge(name, dtype):
    """bik_track_coll with a mask and distances per instance and frame equals one bik_converge_coll per frame, bit for bit,
    with ragged lengths, frames without any pair, and a NaN distance flagged on its frame only."""
    c = _case(name, dtype, B=64 + 5, T=3, seed=12)
    B, T, npairs = c["B"], c["T"], c["npairs"]
    rng = np.random.default_rng(13)
    mask = _random_masks(rng, B * T, npairs, 0.5).reshape(B, T, npairs)
    mask[::4, 1] = False
    dmin, ddet = (x.reshape(B, T) for x in _random_distances(rng, c["lim"], B * T, dtype))
    dmin[5, 2] = np.nan
    ln = _lengths(B, T, 2)
    d = c["d"]
    q = c["dev"](c["q0"])
    q_loop = torch.zeros((B, T, c["fm"].nq), dtype=q.dtype, device=q.device)
    it_loop = torch.zeros((B, T), dtype=torch.int32, device=q.device)
    st_loop = torch.zeros_like(it_loop)
    for t in range(T):
        _, it_loop[:, t], st_loop[:, t] = _converge(c, _dcoll(c, (mask[:, t], dmin[:, t], ddet[:, t])), t=t, q=q)
        q_loop[:, t] = q
    q1 = c["dev"](c["q0"])
    q_traj, it, st, _ = c["prob"].track(q1, d["ft"], d["pt"], d["ct"], lengths=ln, collision=_dcoll(c, (mask, dmin, ddet)), **c["kw"], **CONV)
    has = torch.as_tensor(np.arange(T)[None, :] < ln[:, None], device=q.device)
    _equal(q_traj[has], q_loop[has]); _equal(it[has], it_loop[has]); _equal(st[has], st_loop[has])
    if ln[5] == T:
        assert int(st[5, 2]) & NONFINITE and not (st[5, :2] & NONFINITE).any()


@pytest.mark.parametrize("dtype", [np.float32, np.float64], ids=["f32", "f64"])
def test_nonfinite_distances_are_flagged(dtype):
    """A NaN or infinite distance falls back to the problem's value and sets BIK_STATUS_NONFINITE on that instance only."""
    c = _case("spot", dtype, B=6, T=1, seed=61)
    B, lim = c["B"], c["lim"]
    dmin, ddet = np.full(B, lim.minimum_distance), np.full(B, lim.detection_distance)
    dmin[1], ddet[2], dmin[4] = np.nan, np.inf, -np.inf
    q, it, st = _converge(c, _dcoll(c, (None, dmin, ddet)))
    q_n, it_n, st_n = _converge(c)
    _equal(q, q_n); _equal(it, it_n)
    flag = torch.zeros(B, dtype=torch.int32, device="cuda:0")
    flag[[1, 2, 4]] = NONFINITE
    _equal(st, st_n | flag)


def test_cached_graph_follows_the_collision_buffers():
    """Converge calls on one problem alternating between collision buffers, then the call without them, give what a problem
    without a cached graph gives; so does rewriting a mask in place between two calls."""
    c = _case("ur5e_wall", np.float32, B=256 + 7, T=1, seed=30)
    B, npairs = c["B"], c["npairs"]
    rng = np.random.default_rng(31)
    ca = _dcoll(c, (_random_masks(rng, B, npairs, 0.5), None, None))
    cb = _dcoll(c, (_random_masks(rng, B, npairs, 0.5), *_random_distances(rng, c["lim"], B, np.float32)))
    cc = (ca[0], cb[1], None)
    fresh = lambda co: _converge(c, co, prob=_problem(c["fm"], c["spec"]))
    ref_a, ref_b, ref_c, ref_0 = fresh(ca), fresh(cb), fresh(cc), fresh(None)
    for co, ref in ((ca, ref_a), (cb, ref_b), (ca, ref_a), (None, ref_0), (cc, ref_c), (cb, ref_b)):
        for x, y in zip(_converge(c, co), ref):
            _equal(x, y)
    cb[0].copy_(ca[0])
    ref_ab = fresh((ca[0], cb[1], cb[2]))
    for x, y in zip(_converge(c, cb), ref_ab):
        _equal(x, y)


def test_c_abi_rejects_collision_without_the_limit():
    """A non-null member of bik_collision on a problem without a CollisionAvoidanceLimit: BIK_ERR_INVALID; all-null members
    on such a problem are the ..._bounded call."""
    import ctypes as C

    from mink_b200 import _lib
    from mink_b200._abi import LIMIT_COLLISION, BikCollision

    c = _case("ur5e_wall", np.float32, B=4, T=1, seed=1)
    spec = c["spec"]
    nocoll = type(spec)(spec.tasks, [l for l in spec.limits if l.kind != LIMIT_COLLISION])
    prob = _problem(c["fm"], nocoll)
    d = c["d"]
    junk = torch.ones((4, 8), dtype=torch.float32, device="cuda:0")
    for field in ("enabled", "minimum_distance", "detection_distance"):
        q = c["dev"](c["q0"])
        inp, keep, _, _ = prob._inputs(None, d["ft"][:, 0], d["pt"], None, dtype=q.dtype)
        co = BikCollision()
        setattr(co, field, junk.data_ptr())
        it = torch.zeros(4, dtype=torch.int32, device="cuda:0")
        st = torch.zeros(4, dtype=torch.int32, device="cuda:0")
        rc = prob.lib.bik_converge_coll(prob.handle, 4, q.data_ptr(), C.byref(inp), None, None, None, C.byref(co), float(c["kw"]["dt"]),
                                        float(c["kw"]["damping"]), 10, 2e-3, 2e-3, 1, it.data_ptr(), st.data_ptr(), None)
        assert rc == -1 and b"CollisionAvoidanceLimit" in _lib.load().bik_last_error()
        if field != "enabled":   # (Problem takes an [B, npairs] mask, which is empty here)
            args = [None, None, None]
            args[("enabled", "minimum_distance", "detection_distance").index(field)] = junk[:, 0]
            with pytest.raises(_lib.BikError):
                prob.converge(q, d["ft"][:, 0], d["pt"], None, collision=tuple(args), **c["kw"])
    q = c["dev"](c["q0"])
    q2 = q.clone()
    prob.converge(q, d["ft"][:, 0], d["pt"], None, collision=(None, None, None), **c["kw"])
    prob.converge(q2, d["ft"][:, 0], d["pt"], None, **c["kw"])
    _equal(q, q2)


def _ur5e_wall(fm, q, target, pairs=None):
    """The ur5e_wall workload through the front end: one frame task, a posture task, configuration, velocity and collision
    limits (the wrist against the floor and the wall, or `pairs`)."""
    import mink_b200 as mink
    from mink_b200.lie import SE3
    from mink_b200.workloads import WORKLOADS

    wl = WORKLOADS["ur5e_wall"]
    cl = wl["limits"][2]
    cfg = mink.Configuration(fm, q)
    ee = mink.FrameTask("attachment_site", "site", position_cost=1.0, orientation_cost=1.0, lm_damping=1.0)
    ee.set_target(SE3(wxyz_xyz=target))
    post = mink.PostureTask(fm, cost=1e-2)
    post.set_target(np.asarray(fm.qpos0, np.float64))
    coll = mink.CollisionAvoidanceLimit(fm, pairs or cl["pairs"], gain=cl["gain"], minimum_distance_from_collisions=cl["minimum_distance"],
                                        collision_detection_distance=cl["detection_distance"], bound_relaxation=cl["bound_relaxation"])
    limits = [mink.ConfigurationLimit(fm, gain=0.95), mink.VelocityLimit(fm, {n: wl["limits"][1]["vmax"] for n in fm.names["joint"] if n}), coll]
    return mink, cfg, [ee, post], limits, coll, float(wl["dt"]), float(wl["damping"])


def test_obstacle_subset_batch():
    """One ur5e_wall problem whose even instances disable every wall pair: through converge_ik those instances equal a
    problem built with the floor pair only, bit for bit, and the odd ones the full problem; through track_ik with the wall
    pairs disabled on the middle frame only, every instance equals per-frame converge_ik calls on those problems."""
    if not torch.cuda.is_available():
        pytest.skip("no CUDA device")
    c = _ccase("ur5e_wall", np.float64, B=16, T=3, seed=70)
    fm, B, T = c["fm"], c["B"], c["T"]
    q0 = torch.tensor(c["q0"], dtype=torch.float64, device="cuda:0")
    targets = c["ft"][:, :, 0]
    conv = dict(max_iters=20, pos_threshold=1e-4, ori_threshold=1e-4)
    mink, cfg, tasks, limits, coll, dt, damping = _ur5e_wall(fm, q0.clone(), targets[:, 0])
    wall = coll.pair_mask(["wall"])
    assert wall.any() and not wall.all()
    mask = np.ones((B, len(wall)), bool)
    mask[0::2] = ~wall
    it, ok = mink.converge_ik(cfg, tasks, dt, damping=damping, limits=limits, collision={coll: {"enabled": mask}}, **conv)
    for b in range(B):
        pairs = [(["wrist_3_link"], ["floor"])] if b % 2 == 0 else None
        mink, cfg1, tasks1, limits1, _, _, _ = _ur5e_wall(fm, q0[b:b + 1].clone(), targets[b:b + 1, 0], pairs)
        it1, ok1 = mink.converge_ik(cfg1, tasks1, dt, damping=damping, limits=limits1, **conv)
        _equal(cfg.q_device[b:b + 1], cfg1.q_device)
        assert int(it[b]) == int(it1[0]) and bool(ok[b]) == bool(ok1[0])
    # track: the wall is gone on frame 1 for every instance
    tmask = np.ones((T, len(wall)), bool)
    tmask[1] = ~wall
    mink, cfg_t, tasks_t, limits_t, coll_t, _, _ = _ur5e_wall(fm, q0.clone(), targets[:, 0])
    q_traj, it_t, ok_t = mink.track_ik(cfg_t, tasks_t, dt, {tasks_t[0]: targets}, damping=damping, limits=limits_t,
                                       collision={coll_t: {"enabled": tmask}}, **conv)
    q = q0.clone()
    for t in range(T):
        pairs = [(["wrist_3_link"], ["floor"])] if t == 1 else None
        mink, cfg1, tasks1, limits1, _, _, _ = _ur5e_wall(fm, q.clone(), targets[:, t], pairs)
        it1, _ = mink.converge_ik(cfg1, tasks1, dt, damping=damping, limits=limits1, **conv)
        q = cfg1.q_device.clone()
        _equal(q_traj[:, t], q)
        assert (it_t[:, t].cpu().numpy() == it1).all()


def test_front_end_collision():
    """solve_ik / converge_ik / track_ik with collision={limit: {...}}: masks [npairs] and [B, npairs] (track: [T, npairs],
    [B, T, npairs]), distances as floats, [B] (track: [T], [B, T]); pair_mask by name and id; wrong keys, shapes, limits
    outside the list and a B = T ambiguity are LimitDefinitionError."""
    from mink_b200.exceptions import LimitDefinitionError

    if not torch.cuda.is_available():
        pytest.skip("no CUDA device")
    c = _ccase("ur5e_wall", np.float64, B=4, T=3, seed=80)
    fm, B, T = c["fm"], c["B"], c["T"]
    q0 = torch.tensor(c["q0"], dtype=torch.float64, device="cuda:0")
    targets = c["ft"][:, :, 0]
    mink, cfg, tasks, limits, coll, dt, damping = _ur5e_wall(fm, q0.clone(), targets[:, 0])
    names = fm.names["geom"]
    np.testing.assert_array_equal(coll.pair_mask(["wall"]), coll.pair_mask([names.index("wall")]))
    np.testing.assert_array_equal(coll.pair_mask(["wall"]), [names[b] == "wall" or names[a] == "wall" for a, b in coll.geom_id_pairs])
    assert coll.pair_mask(["wrist_3_link"]).all() and not coll.pair_mask([]).any()
    with pytest.raises(LimitDefinitionError):
        coll.pair_mask(["no_such_geom"])
    npairs = len(coll.geom_id_pairs)
    dmin = np.float32(np.linspace(0.0, 0.02, B)).astype(np.float64)
    v = mink.solve_ik(cfg, tasks, dt, damping=damping, limits=limits,
                      collision={coll: {"enabled": ~coll.pair_mask(["wall"]), "minimum_distance_from_collisions": dmin}})
    for b in range(B):
        mink, cfg1, tasks1, limits1, coll1, _, _ = _ur5e_wall(fm, q0[b:b + 1].clone(), targets[b:b + 1, 0], [(["wrist_3_link"], ["floor"])])
        coll1.minimum_distance_from_collisions = float(dmin[b])
        _equal(v[b:b + 1], mink.solve_ik(cfg1, tasks1, dt, damping=damping, limits=limits1))
    for value in ({"enabled": np.ones((B, npairs))}, {"collision_detection_distance": 0.2}, {"minimum_distance_from_collisions": dmin},
                  {}):
        mink, cfg, tasks, limits, coll, _, _ = _ur5e_wall(fm, q0.clone(), targets[:, 0])
        mink.converge_ik(cfg, tasks, dt, damping=damping, limits=limits, collision={coll: value}, **CONV)
    for value in ({"enabled": np.ones((T, npairs))}, {"enabled": np.ones((B, T, npairs))}, {"collision_detection_distance": np.full(T, 0.2)},
                  {"minimum_distance_from_collisions": np.full((B, T), 0.01)}):
        mink, cfg, tasks, limits, coll, _, _ = _ur5e_wall(fm, q0.clone(), targets[:, 0])
        q_traj, _, _ = mink.track_ik(cfg, tasks, dt, {tasks[0]: targets}, damping=damping, limits=limits, collision={coll: value}, **CONV)
        assert q_traj.shape == (B, T, fm.nq)
    mink, cfg, tasks, limits, coll, _, _ = _ur5e_wall(fm, q0.clone(), targets[:, 0])
    other = _ur5e_wall(fm, q0.clone(), targets[:, 0])[4]
    for bad, lims in (({coll: {"enabled": np.ones(npairs + 1)}}, limits), ({coll: {"enabled": np.ones((B + 1, npairs))}}, limits),
                      ({coll: {"minimum_distance": 0.1}}, limits), ({coll: np.ones(npairs)}, limits), ({other: {}}, limits),
                      ({coll: {}}, None), ({limits[0]: {}}, limits), ({coll: {"collision_detection_distance": np.ones(B + 1)}}, limits)):
        with pytest.raises(LimitDefinitionError):
            mink.solve_ik(cfg, tasks, dt, damping=damping, limits=lims, collision=bad)
    cfgT = _ur5e_wall(fm, q0[:T].clone(), targets[:T, 0])[1]
    with pytest.raises(LimitDefinitionError):   # [3, npairs] with B = T = 3: per instance or per frame?
        mink.track_ik(cfgT, tasks, dt, {tasks[0]: targets[:T]}, damping=damping, limits=limits, collision={coll: {"enabled": np.ones((T, npairs))}})
