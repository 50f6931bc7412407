"""Per-instance joint limits on the device: bik_step_bounded / bik_converge_bounded / bik_track_bounded (and their fp64 forms)
through Problem.step / converge / track, and the `bounds=` mapping of solve_ik / converge_ik / track_ik.

The checks of tests/test_bounds_cpu.py, on the device and on the same cases, with the general K2 also forced by
BIK_K2_PATH=dense: the problem's own bounds give the ..._weighted_ex entry points bit for bit, random narrowing gives a problem
built with the narrowed bounds bit for bit, bik_track_bounded is one bounded converge per frame.  Then
the cached converge graph following the bound buffers, the C ABI's refusals, a TidyBot batch whose base is fixed on half of the
instances by a cap of 0, and the front end.
"""

import numpy as np
import pytest

torch = pytest.importorskip("torch")
pytestmark = pytest.mark.gpu

from tests.test_bounds_cpu import CONV, NAMES, _bcase, _narrowed_spec, _random_bounds  # noqa: E402
from tests.test_gpu_posture_weights import _problem  # noqa: E402

DT = {np.float32: torch.float32, np.float64: torch.float64}
DENSE = {"BIK_K2_PATH": "dense"}


def _case(name, dtype, B, T, seed, env=None):
    if not torch.cuda.is_available():
        pytest.skip("no CUDA device")
    c = _bcase(name, dtype, B=B, T=T, seed=seed)
    c["env"] = env
    c["prob"] = _problem(c["fm"], c["spec"], env)
    dev = lambda a: None if a is None else torch.tensor(np.ascontiguousarray(a), dtype=DT[dtype], device="cuda:0")
    c["d"] = dict(ft=dev(c["ft"]), ct=dev(c["ct"]), pt=dev(c["pt"]), pseq=dev(c["pseq"]))
    c["dev"] = dev
    return c


def _at(a, t):
    return None if a is None else a[:, t]


def _dbounds(c, bd):
    return None if bd is None else tuple(c["dev"](x) for x in bd)


def _converge(c, bd=None, prob=None, t=0, q=None, **kw):
    d = c["d"]
    q = c["dev"](c["q0"]) if q is None else q
    it, st = (prob or c["prob"]).converge(q, d["ft"][:, t], d["pt"], _at(d["ct"], t), bounds=bd, **c["kw"], **(kw or CONV))
    return q, it, st


def _equal(a, b):
    torch.testing.assert_close(a, b, rtol=0, atol=0, equal_nan=True)


def _envs(name):
    return [None] if name == "ur5e_wall" else [None, DENSE]


@pytest.mark.parametrize("dtype", [np.float32, np.float64], ids=["f32", "f64"])
@pytest.mark.parametrize("name", NAMES)
def test_problem_bounds_are_the_identity(name, dtype):
    """Bounds equal to the problem's fp32 values or +-inf: bit for bit the ..._weighted_ex entry points (step, converge, track
    with ragged lengths, with posture weights where the case has posture tasks); also on the general path."""
    for env in _envs(name):
        c = _case(name, dtype, B=200 + 3, T=3, seed=3, env=env)
        B, T, P, nv = c["B"], c["T"], c["P"], c["nv"]
        rng = np.random.default_rng(4)
        (lo0, up0), vm0 = c["cfg"], c["vel"]
        pick = lambda v, inf: np.where(rng.uniform(size=(B, nv)) < 0.3, inf, np.broadcast_to(v, (B, nv)))
        has_cfg = np.isfinite(lo0).any()
        bd = _dbounds(c, (pick(lo0, -np.inf) if has_cfg else None, pick(up0, np.inf) if has_cfg else None,
                          pick(vm0, np.inf) if np.isfinite(vm0).any() else None))
        pw = c["dev"](rng.uniform(0.2, 1.0, size=(B, T, P, nv))) if P else None
        d = c["d"]
        for x, y in zip(_converge(c, bd), _converge(c)):
            _equal(x, y)
        q0, q1 = c["dev"](c["q0"]), c["dev"](c["q0"])
        pw0 = None if pw is None else pw[:, 0].contiguous()
        r0 = c["prob"].step(q0, d["ft"][:, 0], d["pt"], _at(d["ct"], 0), **c["kw"], nsteps=3, integrate=True, posture_weights=pw0, bounds=bd)
        r1 = c["prob"].step(q1, d["ft"][:, 0], d["pt"], _at(d["ct"], 0), **c["kw"], nsteps=3, integrate=True, posture_weights=pw0)
        for x, y in zip((q0,) + r0, (q1,) + r1):
            _equal(x, y)
        ln = torch.tensor(np.random.default_rng(5).integers(0, T + 1, size=B), dtype=torch.int32, device="cuda:0")
        q0, q1 = c["dev"](c["q0"]), c["dev"](c["q0"])
        r0 = c["prob"].track(q0, d["ft"], d["pt"], d["ct"], lengths=ln, posture_weights=pw, bounds=bd, **c["kw"], **CONV)
        r1 = c["prob"].track(q1, d["ft"], d["pt"], d["ct"], lengths=ln, posture_weights=pw, **c["kw"], **CONV)
        for x, y in zip((q0,) + r0[:3], (q1,) + r1[:3]):
            _equal(x, y)
        assert int(r0[3]) == int(r1[3])


@pytest.mark.parametrize("dtype", [np.float32, np.float64], ids=["f32", "f64"])
@pytest.mark.parametrize("name", NAMES)
def test_random_narrowing_is_the_rebuilt_problem(name, dtype):
    """Random fp32-representable narrowing: every instance equals, bit for bit, a device problem built with its narrowed
    bounds (step's dq, converge's q, iterations and status); also on the general path."""
    for env in _envs(name):
        c = _case(name, dtype, B=12, T=1, seed=21, env=env)
        B, nv, fm = c["B"], c["nv"], c["fm"]
        bd = _random_bounds(c, dtype, 22, c["q0"])
        full = [np.full((B, nv), f) if x is None else x.astype(np.float64) for x, f in zip(bd, (-np.inf, np.inf, np.inf))]
        dbd = _dbounds(c, bd)
        d = c["d"]
        q, it, st = _converge(c, dbd)
        dq, st1 = c["prob"].step(c["dev"](c["q0"]), d["ft"][:, 0], d["pt"], _at(d["ct"], 0), **c["kw"], bounds=dbd)
        for b in range(B):
            prob_b = _problem(fm, _narrowed_spec(c["spec"], full[0][b], full[1][b], full[2][b]), env)
            sl = slice(b, b + 1)
            qb = c["dev"](c["q0"][sl])
            it_b, st_b = prob_b.converge(qb, d["ft"][sl, 0], None if d["pt"] is None else d["pt"][sl], None if d["ct"] is None else d["ct"][sl, 0],
                                         **c["kw"], **CONV)
            _equal(q[sl], qb); _equal(it[sl], it_b); _equal(st[sl], st_b)
            dq_b, st1_b = prob_b.step(c["dev"](c["q0"][sl]), d["ft"][sl, 0], None if d["pt"] is None else d["pt"][sl],
                                      None if d["ct"] is None else d["ct"][sl, 0], **c["kw"])
            _equal(dq[sl], dq_b); _equal(st1[sl], st1_b)


@pytest.mark.parametrize("dtype", [np.float32, np.float64], ids=["f32", "f64"])
@pytest.mark.parametrize("name", ["g1", "tidybot", "ur5e_wall"])
def test_track_equals_per_frame_converge(name, dtype):
    """bik_track_bounded equals one bik_converge_bounded per frame, bit for bit, with ragged lengths and per-frame posture
    weights where the case has posture tasks."""
    c = _case(name, dtype, B=128 + 5, T=3, seed=12)
    B, T, P, nv = c["B"], c["T"], c["P"], c["nv"]
    bd = _dbounds(c, _random_bounds(c, dtype, 13, c["q0"]))
    pw = c["dev"](np.random.default_rng(14).uniform(0.0, 1.0, size=(B, T, P, nv))) if P else None
    d = c["d"]
    ln_np = np.random.default_rng(2).integers(0, T + 1, size=B).astype(np.int32)
    q = c["dev"](c["q0"])
    q_loop = torch.zeros((B, T, c["fm"].nq), dtype=q.dtype, device=q.device)
    it_loop = torch.zeros((B, T), dtype=torch.int32, device=q.device)
    st_loop = torch.zeros((B, T), dtype=torch.int32, device=q.device)
    for t in range(T):
        it_loop[:, t], st_loop[:, t] = c["prob"].converge(q, d["ft"][:, t], d["pt"], _at(d["ct"], t), bounds=bd, **c["kw"], **CONV,
                                                          posture_weights=None if pw is None else pw[:, t].contiguous())
        q_loop[:, t] = q
    q_traj, it, st, _ = c["prob"].track(c["dev"](c["q0"]), d["ft"], d["pt"], d["ct"], lengths=torch.tensor(ln_np, device="cuda:0"),
                                        posture_weights=pw, bounds=bd, **c["kw"], **CONV)
    has = torch.tensor(np.arange(T)[None, :] < ln_np[:, None], device="cuda:0")
    _equal(q_traj[has], q_loop[has]); _equal(it[has], it_loop[has]); _equal(st[has], st_loop[has])


def test_cached_graph_follows_the_bound_buffers():
    """Converge calls on one problem alternating between two sets of bound buffers, then the call without bounds, give what a
    problem without a cached graph gives; so does rewriting a buffer in place between two calls."""
    c = _case("g1", np.float32, B=256 + 7, T=1, seed=30)
    ba = _dbounds(c, _random_bounds(c, np.float32, 31, c["q0"]))
    bb = _dbounds(c, _random_bounds(c, np.float32, 32, c["q0"]))
    bc = (ba[0], bb[1], None)
    fresh = lambda bd: _converge(c, bd, prob=_problem(c["fm"], c["spec"]))
    ref_a, ref_b, ref_c, ref_0 = fresh(ba), fresh(bb), fresh(bc), fresh(None)
    for bd, ref in ((ba, ref_a), (bb, ref_b), (ba, ref_a), (None, ref_0), (bc, ref_c), (bb, ref_b)):
        for x, y in zip(_converge(c, bd), ref):
            _equal(x, y)
    for x, y in zip(ba, bb):
        y.copy_(x)
    for x, y in zip(_converge(c, bb), ref_a):
        _equal(x, y)


def test_c_abi_rejects_bounds_without_the_limit():
    """lower / upper on a problem without a ConfigurationLimit, vmax on one without a VelocityLimit: BIK_ERR_INVALID."""
    import ctypes as C

    from mink_b200 import _lib
    from mink_b200._abi import LIMIT_VELOCITY, BikBounds

    c = _case("tidybot", np.float32, B=4, T=1, seed=1)
    spec = c["spec"]
    nocfg = type(spec)(spec.tasks, [l for l in spec.limits if l.kind == LIMIT_VELOCITY])
    novel = type(spec)(spec.tasks, [l for l in spec.limits if l.kind != LIMIT_VELOCITY])
    d = c["d"]
    junk = torch.zeros((4, c["nv"]), dtype=torch.float32, device="cuda:0")
    for sp, field in ((nocfg, "lower"), (nocfg, "upper"), (novel, "vmax")):
        prob = _problem(c["fm"], sp)
        q = c["dev"](c["q0"])
        inp, keep, _, _ = prob._inputs(None, d["ft"][:, 0], d["pt"], None, dtype=q.dtype)
        bd = BikBounds()
        setattr(bd, field, junk.data_ptr())
        it = torch.zeros(4, dtype=torch.int32, device="cuda:0")
        st = torch.zeros(4, dtype=torch.int32, device="cuda:0")
        rc = prob.lib.bik_converge_bounded(prob.handle, 4, q.data_ptr(), C.byref(inp), None, None, C.byref(bd), float(c["kw"]["dt"]),
                                           float(c["kw"]["damping"]), 10, 2e-3, 2e-3, 1, it.data_ptr(), st.data_ptr(), None)
        assert rc == -1 and b"bounds" in _lib.load().bik_last_error()
        args = [None, None, None]
        args[("lower", "upper", "vmax").index(field)] = junk
        with pytest.raises(_lib.BikError):
            prob.converge(q, d["ft"][:, 0], d["pt"], None, bounds=tuple(args), **c["kw"])
    # all-null bounds on those problems are the ..._weighted_ex call
    prob = _problem(c["fm"], nocfg)
    q = c["dev"](c["q0"])
    prob.converge(q, d["ft"][:, 0], d["pt"], None, bounds=(None, None, None), **c["kw"])


def _tidybot(fm, q, target, base_vmax=None):
    """The reference's mobile TidyBot example (examples/mobile_tidybot.py) with a VelocityLimit on the base's three joints."""
    import mink_b200 as mink
    from mink_b200.lie import SE3

    cfg = mink.Configuration(fm, q)
    ee = mink.FrameTask("pinch_site", "site", position_cost=1.0, orientation_cost=1.0, lm_damping=1.0)
    ee.set_target(SE3(wxyz_xyz=target))
    post = mink.PostureTask(fm, cost=np.array([0.0] * 3 + [1e-3] * 15))
    post.set_target(np.asarray(fm.key("home"), np.float64))
    vel = mink.VelocityLimit(fm, base_vmax or {"joint_x": 0.5, "joint_y": 0.5, "joint_th": 1.0})
    return mink, cfg, [ee, post], [mink.ConfigurationLimit(fm, gain=0.95), vel], vel


@pytest.mark.parametrize("dtype", [np.float64, np.float32], ids=["f64", "f32"])
def test_tidybot_fixed_base_batch(dtype):
    """One TidyBot problem, base cap 0 on even instances and no narrowing on odd ones, through converge_ik and track_ik: the
    fixed bases do not move, bit for bit, and every instance equals a separate problem with (even) or without (odd) the zero
    base cap, bit for bit."""
    from tests.helpers import load_case
    from tests.test_posture_weights_cpu import _case as _emu_case

    if not torch.cuda.is_available():
        pytest.skip("no CUDA device")
    wl, fm, spec, g = load_case("tidybot")
    dt, damping = float(wl["dt"]), float(wl["damping"])
    B, T = 16, 3
    c = _emu_case("tidybot", np.float64, B=B, T=T, seed=40)
    q0 = torch.tensor(c["q0"], dtype=DT[dtype], device="cuda:0")
    targets = c["ft"][:, 0, 0]
    vm = np.full((B, 3), np.inf)
    vm[0::2] = 0.0
    conv = dict(max_iters=20, pos_threshold=1e-4, ori_threshold=1e-4)
    mink, cfg, tasks, limits, vel = _tidybot(fm, q0.clone(), targets)
    it, ok = mink.converge_ik(cfg, tasks, dt, damping=damping, limits=limits, bounds={vel: vm}, **conv)
    q = cfg.q_device.clone()
    _equal(q[0::2, :3], q0[0::2, :3])
    assert (q[1::2, :3] != q0[1::2, :3]).any()
    seq = c["ft"][:, :, 0]
    mink, cfg_t, tasks_t, limits_t, vel_t = _tidybot(fm, q0.clone(), targets)
    q_traj, it_t, ok_t = mink.track_ik(cfg_t, tasks_t, dt, {tasks_t[0]: seq}, damping=damping, limits=limits_t, bounds={vel_t: vm}, **conv)
    _equal(q_traj[0::2, :, :3], q0[0::2, None, :3].expand(-1, T, -1))
    for b in range(B):
        fixed = {"joint_x": 0.0, "joint_y": 0.0, "joint_th": 0.0} if b % 2 == 0 else None
        mink, cfg1, tasks1, limits1, _ = _tidybot(fm, q0[b:b + 1].clone(), targets[b:b + 1], fixed)
        it1, ok1 = mink.converge_ik(cfg1, tasks1, dt, damping=damping, limits=limits1, **conv)
        _equal(cfg.q_device[b:b + 1], cfg1.q_device)
        assert int(it[b]) == int(it1[0]) and bool(ok[b]) == bool(ok1[0])
        mink, cfg1, tasks1, limits1, _ = _tidybot(fm, q0[b:b + 1].clone(), targets[b:b + 1], fixed)
        q_traj1, it_t1, _ = mink.track_ik(cfg1, tasks1, dt, {tasks1[0]: seq[b:b + 1]}, damping=damping, limits=limits1, **conv)
        _equal(q_traj[b:b + 1], q_traj1)
        _equal(it_t[b:b + 1], it_t1)


def test_front_end_bounds():
    """solve_ik / converge_ik / track_ik with bounds={limit: value}: [nq] and [B, nq] (ConfigurationLimit), [k] and [B, k]
    (VelocityLimit), None entries; wrong shapes, keys outside the list (the implicit default included), other limit kinds and
    a ConfigurationLimit sharing dofs with another are LimitDefinitionError."""
    import mink_b200 as mink
    from mink_b200.exceptions import LimitDefinitionError
    from mink_b200.lie import SE3
    from tests.helpers import load_case

    if not torch.cuda.is_available():
        pytest.skip("no CUDA device")
    wl, fm, spec, g = load_case("ur5e")
    dt, damping = float(g["dt"]), float(g["damping"])
    B, T, nq = 4, 3, fm.nq
    names = fm.names["joint"]

    def api(q, lower=None, upper=None, vmax=None):
        cfg = mink.Configuration(fm, q)
        ee = mink.FrameTask("attachment_site", "site", position_cost=1.0, orientation_cost=1.0, lm_damping=1.0)
        ee.set_target(SE3(wxyz_xyz=g["frame_targets"][0, 0]))
        post = mink.PostureTask(fm, cost=1e-2)
        post.set_target(g["posture_target"])
        cl = mink.ConfigurationLimit(fm, gain=0.95)
        if lower is not None:
            cl.lower, cl.upper = lower, upper
        vl = mink.VelocityLimit(fm, {n: (1.0 if vmax is None else vmax[i]) for i, n in enumerate(names)})
        return cfg, [ee, post], [cl, vl], cl, vl

    qb = torch.tensor(g["q"][:B], dtype=torch.float64, device="cuda:0")
    rng = np.random.default_rng(1)
    cl0 = api(qb)[3]
    lo = np.float32(np.maximum(cl0.lower, g["q"][:B] - rng.uniform(0.05, 0.5, (B, nq)))).astype(np.float64)
    up = np.float32(np.minimum(cl0.upper, g["q"][:B] + rng.uniform(0.05, 0.5, (B, nq)))).astype(np.float64)
    vm = np.float32(rng.uniform(0.0, 1.0, (B, len(names)))).astype(np.float64)
    cfg, tasks, limits, cl, vl = api(qb.clone())
    v = mink.solve_ik(cfg, tasks, dt, damping=damping, limits=limits, bounds={cl: (lo, up), vl: vm})
    for b in range(B):
        cfg1, tasks1, limits1, _, _ = api(qb[b:b + 1].clone(), np.maximum(np.float32(cl0.lower), lo[b]), np.minimum(np.float32(cl0.upper), up[b]), vm[b])
        _equal(v[b:b + 1], mink.solve_ik(cfg1, tasks1, dt, damping=damping, limits=limits1))
        cfg2, tasks2, limits2, cl2, vl2 = api(qb[b:b + 1].clone())
        _equal(v[b:b + 1], mink.solve_ik(cfg2, tasks2, dt, damping=damping, limits=limits2, bounds={cl2: (lo[b], up[b]), vl2: vm[b]}))
    for bd in ({cl: (lo, None)}, {cl: (None, up)}, {vl: vm[0]}):
        mink.converge_ik(api(qb.clone())[0], tasks, dt, damping=damping, limits=limits, bounds=bd, **CONV)
    seq = np.repeat(g["frame_targets"][0, 0][None], T, axis=0)
    cfg, tasks, limits, cl, vl = api(qb.clone())
    q_traj, iters, ok = mink.track_ik(cfg, tasks, dt, {tasks[0]: seq}, damping=damping, limits=limits, bounds={cl: (lo, up), vl: vm}, **CONV)
    assert q_traj.shape == (B, T, nq)

    cfg, tasks, limits, cl, vl = api(qb.clone())
    other = mink.ConfigurationLimit(fm, gain=0.5)
    for bad, lims in (({cl: (np.ones(nq + 1), None)}, limits), ({cl: (np.ones((B + 1, nq)), None)}, limits), ({vl: np.ones(len(names) + 1)}, limits),
                      ({cl: lo}, limits), ({other: (lo, up)}, limits), ({cl: (lo, up)}, None), ({cl: (lo, up)}, limits + [other]),
                      ({tasks[1]: (lo, up)}, limits)):
        with pytest.raises(LimitDefinitionError):
            mink.solve_ik(cfg, tasks, dt, damping=damping, limits=lims, bounds=bad)
    mink.solve_ik(cfg, tasks, dt, damping=damping, limits=limits + [other], bounds={vl: vm})   # only a ConfigurationLimit key is ambiguous
