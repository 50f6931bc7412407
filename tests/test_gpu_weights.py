"""Per-instance task weights on the device: bik_step_weighted / bik_converge_weighted / bik_track_weighted (and their fp64
forms) through Problem.step / converge / track, and the `weights=` mapping of solve_ik / converge_ik / track_ik.

All-ones weights give the unweighted entry points' results bit for bit; instance b with weights w[b] solves what the fp64
oracle solves with the costs cost * w[b]; zero weights on a frame task remove it; out-of-range weights are clamped and
flagged with BIK_STATUS_BAD_WEIGHT.  bik_track_weighted keeps bik_track's contract: bit for bit one
bik_converge_weighted call per frame on the same buffers.
"""

import numpy as np
import pytest

torch = pytest.importorskip("torch")
pytestmark = pytest.mark.gpu

from tests.helpers import load_case, track_case  # noqa: E402
from tests.test_weights_cpu import BAD_WEIGHT, _row_blocks, _weighted_spec, _without_task  # noqa: E402

CONV = dict(max_iters=10, pos_threshold=2e-3, ori_threshold=2e-3)
DT = {np.float32: torch.float32, np.float64: torch.float64}


def _need_gpu():
    if not torch.cuda.is_available():
        pytest.skip("no CUDA device")


def _case(name, B, T, seed, dtype, sigma=0.3, spec=None):
    """track_case's targets as CUDA tensors of `dtype`, with a device Problem (of `spec`, default the workload's)."""
    _need_gpu()
    from mink_b200.engine import DeviceModel, Problem

    c = track_case(name, B=B, T=T, seed=seed, dtype=dtype, sigma=sigma)
    wl, fm, spec0, g = load_case(name)
    c["fm"], c["spec"] = fm, spec if spec is not None else spec0
    c["prob"] = Problem(DeviceModel(fm, device=0), c["spec"])
    dev = lambda a: None if a is None else torch.tensor(np.ascontiguousarray(a), dtype=DT[dtype], device="cuda:0")
    c["d"] = dict(ft=dev(c["ft"]), ct=dev(c["ct"]), pt=dev(c["pt"]))
    c["dev"], c["dtype"] = dev, dtype
    return c


def _frame(c, t):
    d = c["d"]
    return d["ft"][:, t], d["pt"], None if d["ct"] is None else d["ct"][:, t]


def _converge(c, w=None, t=0, q=None, **kw):
    q = c["dev"](c["q0"]) if q is None else q
    it, st = c["prob"].converge(q, *_frame(c, t), weights=w, **c["kw"], **(kw or CONV))
    return q, it, st


def _equal(a, b):
    torch.testing.assert_close(a, b, rtol=0, atol=0, equal_nan=True)


@pytest.mark.parametrize("dtype", [np.float32, np.float64])
@pytest.mark.parametrize("name", ["ur5e", "g1", "spot"])
def test_ones_are_the_identity(name, dtype):
    c = _case(name, B=200 + 3, T=4, seed=3, dtype=dtype)
    B, T, K = c["B"], c["T"], c["spec"].nrows
    ones = torch.ones((B, K), dtype=DT[dtype], device="cuda:0")
    for x, y in zip(_converge(c, ones), _converge(c)):
        _equal(x, y)
    q0, q1 = c["dev"](c["q0"]), c["dev"](c["q0"])
    r0 = c["prob"].step(q0, *_frame(c, 0), **c["kw"], nsteps=3, integrate=True, weights=ones)
    r1 = c["prob"].step(q1, *_frame(c, 0), **c["kw"], nsteps=3, integrate=True)
    for x, y in zip((q0,) + r0, (q1,) + r1):
        _equal(x, y)
    d = c["d"]
    ln = torch.tensor(np.random.default_rng(4).integers(0, T + 1, size=B), dtype=torch.int32, device="cuda:0")
    q0, q1 = c["dev"](c["q0"]), c["dev"](c["q0"])
    r0 = c["prob"].track(q0, d["ft"], d["pt"], d["ct"], lengths=ln, weights=torch.ones((B, T, K), dtype=DT[dtype], device="cuda:0"),
                         **c["kw"], **CONV)
    r1 = c["prob"].track(q1, d["ft"], d["pt"], d["ct"], lengths=ln, **c["kw"], **CONV)
    for x, y in zip((q0,) + r0[:3], (q1,) + r1[:3]):
        _equal(x, y)
    assert int(r0[3]) == int(r1[3])


@pytest.mark.parametrize("dtype", [np.float64, np.float32])
@pytest.mark.parametrize("name", ["ur5e", "g1", "spot"])
def test_weights_are_costs(name, dtype):
    """bik_step_weighted's dq and one bik_converge_weighted step against the fp64 oracle with the costs cost * w[b]: 1e-8 rad
    in fp64, 1e-4 rad in fp32."""
    from oracle.ikoracle import Oracle

    c = _case(name, B=8, T=1, seed=21, dtype=dtype)
    fm, spec, B, K = c["fm"], c["spec"], c["B"], c["spec"].nrows
    w = np.random.default_rng(5).uniform(0.1, 1.0, size=(B, K)).astype(dtype)
    wd = c["dev"](w)
    dq, st = c["prob"].step(c["dev"](c["q0"]), *_frame(c, 0), **c["kw"], weights=wd)
    q1, _, st1 = _converge(c, wd, max_iters=1, pos_threshold=0.0, ori_threshold=0.0)
    assert not st.any() and not (st1 & ~16).any()
    dq, q1 = dq.cpu().numpy(), q1.cpu().numpy()
    f64 = lambda a: None if a is None else np.asarray(a, np.float64)
    tol = 1e-8 if dtype == np.float64 else 1e-4
    for b in range(B):
        orc = Oracle(fm.to_blob(), _weighted_spec(spec, w[b].astype(np.float64)), fm.nq, fm.nv)
        ct = None if c["ct"] is None else f64(c["ct"][b:b + 1, 0])
        dq_ref, q_ref, st_ref, _ = orc.step(f64(c["q0"][b:b + 1]), f64(c["ft"][b:b + 1, 0]), f64(c["pt"][b:b + 1]), ct, **c["kw"],
                                            nsteps=1, integrate=True)
        assert not st_ref.any()
        np.testing.assert_allclose(dq[b], dq_ref[0], atol=tol, rtol=0)
        np.testing.assert_allclose(q1[b], q_ref[0], atol=tol, rtol=0)


@pytest.mark.parametrize("dtype", [np.float64, np.float32])
def test_zero_weights_remove_the_task(dtype):
    """G1's right foot weighted 0 (its target 0.3 m away): the problem without that task, with the same iteration counts."""
    c = _case("g1", B=256, T=1, seed=8, dtype=dtype, sigma=0.1)
    spec, B, K = c["spec"], c["B"], c["spec"].nrows
    _, (i1, r1, _), _ = _row_blocks(spec)
    c["d"]["ft"][:, :, 1, 4:] += 0.3
    w = torch.ones((B, K), dtype=DT[dtype], device="cuda:0")
    w[:, r1:r1 + 6] = 0.0
    conv = dict(max_iters=15, pos_threshold=1e-2, ori_threshold=1e-2)
    q, it, st = _converge(c, w, **conv)
    s = _case("g1", B=256, T=1, seed=8, dtype=dtype, sigma=0.1, spec=_without_task(spec, i1))
    s["d"]["ft"] = torch.cat([c["d"]["ft"][:, :, :1], c["d"]["ft"][:, :, 2:]], dim=2).contiguous()
    q_s, it_s, st_s = _converge(s, **conv)
    tol = 1e-9 if dtype == np.float64 else 1e-5
    assert (q - q_s).abs().max().item() <= tol
    _equal(it, it_s)
    _equal(st, st_s)
    assert (it < conv["max_iters"]).any()


@pytest.mark.parametrize("dtype", [np.float32, np.float64])
def test_out_of_range_and_nan_weights_are_clamped_and_flagged(dtype):
    c = _case("spot", B=64, T=1, seed=9, dtype=dtype)
    B, K = c["B"], c["spec"].nrows
    w = np.random.default_rng(10).uniform(0.2, 1.0, size=(B, K)).astype(dtype)
    bad, clamped = w.copy(), w.copy()
    bad[1, 0], clamped[1, 0] = 1.5, 1.0
    bad[4, 7], clamped[4, 7] = -0.25, 0.0
    bad[7, K - 1], clamped[7, K - 1] = np.nan, 0.0
    flagged = np.zeros(B, np.int32)
    flagged[[1, 4, 7]] = BAD_WEIGHT
    q, it, st = _converge(c, c["dev"](bad))
    q_c, it_c, st_c = _converge(c, c["dev"](clamped))
    _equal(q, q_c)
    _equal(it, it_c)
    assert not (st_c & BAD_WEIGHT).any()
    np.testing.assert_array_equal(st.cpu().numpy(), st_c.cpu().numpy() | flagged)
    _, st = c["prob"].step(c["dev"](c["q0"]), *_frame(c, 0), **c["kw"], weights=c["dev"](bad))
    assert ((st.cpu().numpy() & BAD_WEIGHT) == flagged).all()


@pytest.mark.parametrize("dtype", [np.float32, np.float64])
@pytest.mark.parametrize("name", ["ur5e", "h1"])
def test_track_weighted_equals_per_frame_converge_weighted(name, dtype):
    """[B][T][K] weights: bik_track_weighted is bit for bit one bik_converge_weighted call per frame on the same q, with
    ragged lengths; half the instances have a frame task fully weighted 0 on some frames."""
    c = _case(name, B=300 + 5, T=5, seed=12, dtype=dtype)
    B, T, K = c["B"], c["T"], c["spec"].nrows
    rng = np.random.default_rng(13)
    w = rng.uniform(0.0, 1.0, size=(B, T, K)).astype(dtype)
    occluded = rng.random((B, T)) < 0.5
    w[:, :, :6][occluded] = 0.0
    wd = c["dev"](w)
    ln = np.random.default_rng(2).integers(0, T + 1, size=B).astype(np.int32)
    q = c["dev"](c["q0"])
    q_loop = torch.zeros((B, T, c["fm"].nq), dtype=q.dtype, device="cuda:0")
    it_loop = torch.zeros((B, T), dtype=torch.int32, device="cuda:0")
    st_loop = torch.zeros((B, T), dtype=torch.int32, device="cuda:0")
    for t in range(T):
        _, it_loop[:, t], st_loop[:, t] = _converge(c, wd[:, t].contiguous(), t=t, q=q)
        q_loop[:, t] = q
    d = c["d"]
    q_end = c["dev"](c["q0"])
    q_traj, it, st, _ = c["prob"].track(q_end, d["ft"], d["pt"], d["ct"], lengths=torch.tensor(ln, device="cuda:0"), weights=wd,
                                        **c["kw"], **CONV)
    has = torch.tensor(np.arange(T)[None, :] < ln[:, None], device="cuda:0")
    _equal(q_traj[has], q_loop[has])
    _equal(it[has], it_loop[has])
    _equal(st[has], st_loop[has])


def test_cached_graph_follows_the_weights_buffer():
    """A second weighted converge call on the same problem with another weights buffer, then a larger batch, gives what a
    problem without a cached graph gives."""
    c = _case("ur5e", B=256 + 7, T=1, seed=30, dtype=np.float32)
    B, K = c["B"], c["spec"].nrows
    rng = np.random.default_rng(31)
    wa, wb = (c["dev"](rng.uniform(0.0, 1.0, size=(B, K)).astype(np.float32)) for _ in range(2))
    fresh = lambda w: _converge(dict(c, prob=_case("ur5e", B=8, T=1, seed=0, dtype=np.float32)["prob"]), w)
    ref_a, ref_b = fresh(wa), fresh(wb)
    for w, ref in ((wa, ref_a), (wb, ref_b), (wa, ref_a)):
        for x, y in zip(_converge(c, w), ref):
            _equal(x, y)
    big = _case("ur5e", B=2 * B, T=1, seed=30, dtype=np.float32)
    wbig = torch.cat([wb, wa])
    ref = _converge(dict(big, prob=_case("ur5e", B=8, T=1, seed=0, dtype=np.float32)["prob"]), wbig)
    for x, y in zip(_converge(dict(big, prob=c["prob"]), wbig), ref):
        _equal(x, y)


def _ur5e_api(g, fm, b, pos_cost=1.0, ori_cost=1.0, q=None):
    import mink_b200 as mink
    from mink_b200.lie import SE3

    cfg = mink.Configuration(fm, g["q"][b] if q is None else q)
    ee = mink.FrameTask("attachment_site", "site", position_cost=pos_cost, orientation_cost=ori_cost, lm_damping=1.0)
    ee.set_target(SE3(wxyz_xyz=g["frame_targets"][b, 0]))
    post = mink.PostureTask(fm, cost=1e-2)
    post.set_target(g["posture_target"])
    return mink, cfg, ee, [ee, post], [mink.ConfigurationLimit(fm, gain=0.95)]


def test_front_end_weights():
    """solve_ik / converge_ik / track_ik with weights={task: w}: a single (fp64) configuration equals the problem with the
    task's costs multiplied by w; batches take [B, 6], [T, 6] and [B, T, 6]; wrong shapes and PostureTask keys are
    InvalidTarget; a bad weight fails the solve."""
    from mink_b200.exceptions import InvalidTarget

    _need_gpu()
    wl, fm, spec, g = load_case("ur5e")
    dt, damping = float(g["dt"]), float(g["damping"])
    w = np.array([0.5, 0.25, 1.0, 0.75, 0.5, 0.125])   # exact in fp32, like the costs the problem image holds
    for b in range(3):
        mink, cfg, ee, tasks, limits = _ur5e_api(g, fm, b)
        v = mink.solve_ik(cfg, tasks, dt, damping=damping, limits=limits, weights={ee: w})
        mink, cfg2, ee2, tasks2, limits2 = _ur5e_api(g, fm, b, pos_cost=w[:3], ori_cost=w[3:])
        v_ref = mink.solve_ik(cfg2, tasks2, dt, damping=damping, limits=limits2)
        assert isinstance(v, np.ndarray) and v.dtype == np.float64
        np.testing.assert_array_equal(v, v_ref)
        it, ok = mink.converge_ik(cfg, tasks, dt, damping=damping, limits=limits, weights={ee: w}, **CONV)
        it2, ok2 = mink.converge_ik(cfg2, tasks2, dt, damping=damping, limits=limits2, **CONV)
        assert (it, ok) == (it2, ok2)
        np.testing.assert_array_equal(cfg.q, cfg2.q)

    B, T = 4, 3
    qb = torch.tensor(g["q"][:B], dtype=torch.float32, device="cuda:0")
    mink, cfg, ee, tasks, limits = _ur5e_api(g, fm, 0, q=qb.clone())
    wb = np.random.default_rng(1).uniform(0.2, 1.0, size=(B, 6))
    v = mink.solve_ik(cfg, tasks, dt, damping=damping, limits=limits, weights={ee: wb})
    for b in range(B):
        _, cfg1, ee1, tasks1, limits1 = _ur5e_api(g, fm, 0, q=qb[b:b + 1].clone())
        v1 = mink.solve_ik(cfg1, tasks1, dt, damping=damping, limits=limits1, weights={ee1: wb[b]})
        _equal(v[b:b + 1], v1)
    seq = np.repeat(g["frame_targets"][0, 0][None], T, axis=0)
    for ws in (wb[0], wb[:T], np.broadcast_to(wb[:, None], (B, T, 6))):
        _, cfg, ee, tasks, limits = _ur5e_api(g, fm, 0, q=qb.clone())
        q_traj, iters, ok = mink.track_ik(cfg, tasks, dt, {ee: seq}, damping=damping, limits=limits, weights={ee: ws}, **CONV)
        assert q_traj.shape == (B, T, fm.nq) and (iters >= 1).all()

    _, cfg, ee, tasks, limits = _ur5e_api(g, fm, 0, q=qb.clone())
    for bad in ({ee: np.ones(3)}, {ee: np.ones((B + 1, 6))}, {tasks[1]: np.ones(fm.nv)}):
        with pytest.raises(InvalidTarget):
            mink.solve_ik(cfg, tasks, dt, damping=damping, limits=limits, weights=bad)
    with pytest.raises(InvalidTarget):
        mink.track_ik(cfg, tasks, dt, {ee: seq}, damping=damping, limits=limits, weights={ee: np.ones((T + 1, 6))})
    with pytest.raises(AssertionError):
        mink.solve_ik(cfg, tasks, dt, damping=damping, limits=limits, weights={ee: np.full(6, np.nan)})
