"""bik_converge64 / bik_track64 / Problem.converge and Problem.track on float64 q / converge_ik and track_ik in fp64.

The fp64 loops keep the reference's precision end to end: iteration counts and flags equal to the goldens and to the C
oracle's loop, final configurations within the oracle's own bars.  bik_track64 gives bit for bit what T calls of
bik_converge64 give, as bik_track does for bik_converge.
"""

import ctypes as C
import os

import numpy as np
import pytest

torch = pytest.importorskip("torch")
pytestmark = pytest.mark.gpu

from mink_b200.workloads import make_inputs  # noqa: E402
from tests.helpers import load_case, task_frames  # noqa: E402

CASES = ["ur5e", "ur5e_dls", "g1", "shadow", "spot", "g1_rel", "edge", "g1_full", "g1_hands", "ur5e_damp", "ur5e_wall",
         "iiwa", "h1", "go1", "stretch", "tidybot", "aloha", "aloha_coll", "leap"]
GOLDEN_TOL = {"spot": 1e-3, "g1_rel": 1e-4, "edge": 1e-5}            # the oracle's bars (test_converge_loop) times 10
FP32_TOL = {"spot": 1e-2, "edge": 1e-2, "g1_rel": 5e-3}               # bik_converge's bars (test_converge_matches_reference)
CONV = dict(max_iters=10, pos_threshold=2e-3, ori_threshold=2e-3)


def _need_gpu():
    if not torch.cuda.is_available():
        pytest.skip("no CUDA device")


def _engine(name):
    _need_gpu()
    from mink_b200.engine import DeviceModel, Problem

    wl, fm, spec, g = load_case(name)
    model = DeviceModel(fm, device=0)
    return wl, fm, spec, g, model, Problem(model, spec)


def _oracle(fm, spec):
    from oracle.ikoracle import Oracle

    return Oracle(fm.to_blob(), spec, fm.nq, fm.nv)


def _d64(a):
    return None if a is None else torch.tensor(np.ascontiguousarray(a), dtype=torch.float64, device="cuda:0")


def _equal(a, b):
    a, b = a.cpu(), b.cpu()
    assert a.dtype == b.dtype and torch.equal(a, b), f"{int((a != b).sum())} elements differ"


class _graph_mode:
    def __init__(self, mode):
        self.mode = mode

    def __enter__(self):
        os.environ["BIK_CONVERGE_GRAPH"] = self.mode

    def __exit__(self, *a):
        os.environ.pop("BIK_CONVERGE_GRAPH", None)


@pytest.mark.parametrize("name", CASES)
def test_converge64_matches_golden_loops(name):
    wl, fm, spec, g, model, prob = _engine(name)
    CB = g["conv_q"].shape[0]
    max_iters, pos, ori = int(g["conv_params"][0]), float(g["conv_params"][1]), float(g["conv_params"][2])
    ct = g["com_target"][:CB] if "com_target" in g else None
    q = _d64(g["q"][:CB])
    it, st = prob.converge(q, g["frame_targets"][:CB], g["posture_target"], ct, dt=float(g["dt"]), damping=float(g["damping"]),
                           max_iters=max_iters, pos_threshold=pos, ori_threshold=ori)
    sti = st.cpu().numpy().astype(np.int64)
    np.testing.assert_array_equal(it.cpu().numpy(), g["conv_iters"])
    np.testing.assert_array_equal((sti & 16) == 0, g["conv_ok"].astype(bool))
    assert int((sti & 15).max()) == 0
    err = np.abs(q.cpu().numpy() - g["conv_q"]).max()
    print(f"{name}: max|q - q_golden| = {err:.2e}  (fp64 bar {GOLDEN_TOL.get(name, 1e-6):.0e}, fp32 bar {FP32_TOL.get(name, 1e-3):.0e})")
    assert err <= GOLDEN_TOL.get(name, 1e-6)


@pytest.mark.parametrize("check_every", [1, 3])
def test_converge64_batch_against_oracle(check_every):
    """The ragged UR5e batch of test_converge_batch_against_oracle: every iteration count equals the oracle's."""
    wl, fm, spec, g, model, prob = _engine("ur5e")
    orc = _oracle(fm, spec)
    frames = task_frames(wl, fm)
    B = 1500 + 13
    inp = make_inputs(fm, wl, B, lambda qq: orc.fk(qq, frames), seed=5, sigma=0.05)
    q = _d64(inp["q"])
    it, st = prob.converge(q, inp["frame_targets"], inp["posture_target"], None, dt=wl["dt"], damping=wl["damping"], max_iters=12,
                           pos_threshold=2e-3, ori_threshold=2e-3, check_every=check_every)
    q_ref, it_ref, ok_ref, _ = orc.converge(inp["q"], inp["frame_targets"], inp["posture_target"], None, dt=wl["dt"], damping=wl["damping"],
                                            max_iters=12, pos_threshold=2e-3, ori_threshold=2e-3)
    it = it.cpu().numpy()
    print(f"converge64: mismatching iters {int((it != it_ref).sum())}/{B}, max|q - q_oracle| {np.abs(q.cpu().numpy() - q_ref).max():.2e}")
    np.testing.assert_array_equal(it, it_ref)
    np.testing.assert_array_equal((st.cpu().numpy() & 16) == 0, ok_ref.astype(bool))
    np.testing.assert_allclose(q.cpu().numpy(), q_ref, atol=1e-6)


def _case(name, B, T, seed, sigma=0.3):
    wl, fm, spec, g, model, prob = _engine(name)
    orc = _oracle(fm, spec)
    frames = task_frames(wl, fm)
    fk = lambda qq: orc.fk(qq, frames)
    inp = make_inputs(fm, wl, B, fk, seed=seed, sigma=sigma)
    rng = np.random.default_rng(seed + 1)
    path = np.repeat(inp["q"][:, None, :], T, axis=1)
    frac = np.arange(1, T + 1) / T
    for n in range(fm.nnode):
        if int(fm.node_type[n]) >= 2:   # hinge / slide
            path[:, :, int(fm.node_qadr[n])] += rng.normal(0.0, sigma, size=B)[:, None] * frac[None, :]
    poses, com = fk(path.reshape(B * T, fm.nq))
    ft = _d64(np.asarray(poses).reshape(B, T, -1, 7))
    ct = _d64(np.asarray(com).reshape(B, T, -1, 3)) if spec.ncom else None
    pt = _d64(inp["q"][:, None, :])
    return dict(wl=wl, fm=fm, spec=spec, prob=prob, orc=orc, q0=inp["q"], ft=ft, ct=ct, pt=pt,
                kw=dict(dt=wl["dt"], damping=wl["damping"]), B=B, T=T)


def _per_frame(c, dtype=torch.float64, **kw):
    q = torch.tensor(c["q0"], dtype=dtype, device="cuda:0")
    qs, its, sts = [], [], []
    for t in range(c["T"]):
        it, st = c["prob"].converge(q, c["ft"][:, t], c["pt"], None if c["ct"] is None else c["ct"][:, t], **c["kw"], **kw)
        qs.append(q.clone()); its.append(it.clone()); sts.append(st.clone())
    return torch.stack(qs, 1), torch.stack(its, 1), torch.stack(sts, 1), q


def _track(c, dtype=torch.float64, lengths=None, **kw):
    q = torch.tensor(c["q0"], dtype=dtype, device="cuda:0")
    q_traj, it, st, passes = c["prob"].track(q, c["ft"], c["pt"], c["ct"], lengths=lengths, **c["kw"], **kw)
    return q_traj, it, st, q, int(passes)


@pytest.mark.parametrize("mode", ["1", "0"])
@pytest.mark.parametrize("name", ["ur5e", "g1", "h1", "ur5e_wall", "spot"])
def test_track64_equals_the_per_frame_converge64_loop(name, mode):
    """Mixed lengths (0, T and 1 included), graph mode and the host-polled loop (polled every 3 passes)."""
    c = _case(name, B=600 + 13, T=8, seed=21)
    B, T = c["B"], c["T"]
    ln = np.random.default_rng(3).integers(0, T + 1, size=B).astype(np.int32)
    ln[:3] = [0, T, 1]
    with _graph_mode(mode):
        q_loop, it_loop, st_loop, _ = _per_frame(c, check_every=3, **CONV)
        q_traj, it, st, q, passes = _track(c, lengths=torch.tensor(ln, device="cuda:0"), check_every=3, **CONV)
    assert q_traj.dtype == torch.float64
    q_loop, it_loop, st_loop = q_loop.cpu().numpy(), it_loop.cpu().numpy(), st_loop.cpu().numpy()
    q_traj, it, st, q = q_traj.cpu().numpy(), it.cpu().numpy(), st.cpu().numpy(), q.cpu().numpy()
    has = np.arange(T)[None, :] < ln[:, None]
    np.testing.assert_array_equal(q_traj[has], q_loop[has])
    np.testing.assert_array_equal(it[has], it_loop[has])
    np.testing.assert_array_equal(st[has], st_loop[has])
    assert np.isnan(q_traj[~has]).all() and (it[~has] == -1).all() and (st[~has] == -1).all()
    q_ref = np.where(ln[:, None] > 0, q_loop[np.arange(B), np.maximum(ln - 1, 0)], c["q0"])
    np.testing.assert_array_equal(q, q_ref)
    assert passes == int(np.where(has, it + 1, 0).sum(1).max())
    print(f"{name}: iters histogram {np.bincount(it[has]).tolist()} passes {passes}")


def test_converge64_graph_equals_host_polled():
    c = _case("g1", B=700 + 3, T=1, seed=8)
    out = {}
    for mode in ("1", "0"):
        with _graph_mode(mode):
            out[mode] = _per_frame(c, check_every=2, **CONV)
    for x, y in zip(out["1"], out["0"]):
        _equal(x, y)


def test_graph_cache_across_precisions():
    """converge64 -> converge -> track64 -> converge64 -> track on one problem: each call equals the same call made fresh."""
    c = _case("ur5e", B=300 + 5, T=5, seed=55)
    kinds = {
        "converge64": lambda: _per_frame(dict(c, T=1), **CONV),
        "converge": lambda: _per_frame(dict(c, T=1, ft=c["ft"].float(), pt=c["pt"].float()), dtype=torch.float32, **CONV),
        "track64": lambda: _track(c, **CONV)[:4],
        "track": lambda: _track(dict(c, ft=c["ft"].float(), pt=c["pt"].float()), dtype=torch.float32, **CONV)[:4],
    }
    fresh = {}
    for k, f in kinds.items():
        c["prob"] = _case("ur5e", B=300 + 5, T=5, seed=55)["prob"]   # a problem without a cached graph
        fresh[k] = f()
    c["prob"] = _case("ur5e", B=300 + 5, T=5, seed=55)["prob"]
    for k in ("converge64", "converge", "track64", "converge64", "track"):
        for x, y in zip(kinds[k](), fresh[k]):
            _equal(x, y)


def _ur5e_api(b, g, fm):
    import mink_b200 as mink
    from mink_b200.lie import SE3

    cfg = mink.Configuration(fm, g["q"][b])
    ee = mink.FrameTask("attachment_site", "site", position_cost=1.0, orientation_cost=1.0, lm_damping=1.0)
    ee.set_target(SE3(wxyz_xyz=g["frame_targets"][b, 0]))
    post = mink.PostureTask(fm, cost=1e-2)
    post.set_target(g["posture_target"])
    return mink, SE3, cfg, [ee, post], ee, [mink.ConfigurationLimit(fm, gain=0.95)]


def test_converge_ik_single_configuration_equals_the_explicit_fp64_loop():
    wl, fm, spec, g = load_case("ur5e")
    _need_gpu()
    max_iters, pos, ori = int(g["conv_params"][0]), float(g["conv_params"][1]), float(g["conv_params"][2])
    dt, damping = float(g["dt"]), float(g["damping"])
    for b in range(4):
        mink, SE3, cfg, tasks, ee, limits = _ur5e_api(b, g, fm)
        it, ok = mink.converge_ik(cfg, tasks, dt, "quadprog", damping, limits=limits, max_iters=max_iters, pos_threshold=pos,
                                  ori_threshold=ori)
        assert it == int(g["conv_iters"][b]) and ok == bool(g["conv_ok"][b])
        _, _, cfg2, tasks2, ee2, limits2 = _ur5e_api(b, g, fm)
        steps = 0
        for i in range(max_iters):
            v = mink.solve_ik(cfg2, tasks2, dt, "quadprog", damping, limits=limits2)
            cfg2.integrate_inplace(v, dt)
            steps = i + 1
            err = ee2.compute_error(cfg2)
            if np.linalg.norm(err[:3]) <= pos and np.linalg.norm(err[3:]) <= ori:
                break
        print(f"instance {b}: iters {it}, max|q - q_loop| {np.abs(cfg.q - cfg2.q).max():.2e}")
        assert steps == it
        np.testing.assert_allclose(cfg.q, cfg2.q, atol=1e-9)


def test_track_ik_single_configuration_is_fp64():
    """A single configuration: float64 numpy out, bit-equal to converge_ik after set_target on every frame; cfg.q is the last
    row.  A float64 batch: float64 tensors out."""
    wl, fm, spec, g = load_case("ur5e")
    _need_gpu()
    T = 5
    seq = np.repeat(g["frame_targets"][0, 0][None], T, axis=0)   # [T, 7]: the end effector moves 5 cm along x, y and z
    seq[:, 4:] += np.linspace(0.0, 0.05, T)[:, None]
    dt, damping = float(g["dt"]), float(g["damping"])
    mink, SE3, cfg, tasks, ee, limits = _ur5e_api(0, g, fm)
    q_traj, iters, ok = mink.track_ik(cfg, tasks, dt, {ee: seq}, damping=damping, limits=limits, **CONV)
    assert isinstance(q_traj, np.ndarray) and q_traj.dtype == np.float64 and q_traj.shape == (T, fm.nq)
    np.testing.assert_array_equal(cfg.q, q_traj[-1])
    _, _, cfg2, tasks2, ee2, limits2 = _ur5e_api(0, g, fm)
    for t in range(T):
        ee2.set_target(SE3(wxyz_xyz=seq[t]))
        it, okt = mink.converge_ik(cfg2, tasks2, dt, damping=damping, limits=limits2, **CONV)
        np.testing.assert_array_equal(cfg2.q, q_traj[t])
        assert it == int(iters[t]) and okt == bool(ok[t])

    qb = torch.tensor(g["q"][:3], dtype=torch.float64, device="cuda:0")
    cfgb = mink.Configuration(fm, qb)
    ee.set_target(SE3(wxyz_xyz=g["frame_targets"][0, 0]))
    q_traj_b, iters_b, ok_b = mink.track_ik(cfgb, tasks, dt, {ee: seq}, damping=damping, limits=limits, **CONV)
    assert q_traj_b.dtype == torch.float64 and q_traj_b.shape == (3, T, fm.nq)
    assert cfgb.q_device.dtype == torch.float64
    _equal(q_traj_b[:, -1], cfgb.q_device)


def test_converge64_and_track64_errors():
    from mink_b200._lib import BikError, check

    c = _case("ur5e", B=16, T=4, seed=1)
    prob, lib = c["prob"], c["prob"].lib
    st = torch.cuda.current_stream().cuda_stream
    q64 = torch.tensor(c["q0"], dtype=torch.float64, device="cuda:0")
    q32 = q64.float()
    it = torch.zeros((16, 4), dtype=torch.int32, device="cuda:0")
    status = torch.zeros((16, 4), dtype=torch.int32, device="cuda:0")
    qt64 = torch.zeros((16, 4, c["fm"].nq), dtype=torch.float64, device="cuda:0")
    inp32, keep32, _, _ = prob._inputs(None, c["ft"][:, 0], c["pt"], None, dtype=torch.float32)
    inp64, keep64, _, _ = prob._inputs(None, c["ft"][:, 0], c["pt"], None, dtype=torch.float64)
    tin64, tkeep64, _, _ = prob._inputs(None, c["ft"], c["pt"], None, dtype=torch.float64)
    tin32, tkeep32, _, _ = prob._inputs(None, c["ft"], c["pt"], None, dtype=torch.float32)
    conv = lambda fn, q, inp: check(fn(prob.handle, 16, None if q is None else q.data_ptr(), C.byref(inp), 0.01, 1e-12, 10, 2e-3, 2e-3,
                                       1, it.data_ptr(), status.data_ptr(), st))

    def track(fn, q, inp, T=4, lengths=None, qt=qt64):
        return check(fn(prob.handle, 16, T, None if q is None else q.data_ptr(), C.byref(inp), None if lengths is None else lengths.data_ptr(),
                        0.01, 1e-12, 10, 2e-3, 2e-3, 1, qt.data_ptr(), it.data_ptr(), status.data_ptr(), None, st))

    with pytest.raises(BikError, match="f64 must be 1"):
        conv(lib.bik_converge64, q64, inp32)
    with pytest.raises(BikError, match="f64 must be 1"):
        track(lib.bik_track64, q64, tin32)
    with pytest.raises(BikError, match="f64 must be 0"):
        conv(lib.bik_converge, q32, inp64)
    with pytest.raises(BikError, match="f64 must be 0"):
        track(lib.bik_track, q32, tin64)
    for bad in (-1, 5):
        ln = torch.full((16,), 2, dtype=torch.int32, device="cuda:0")
        ln[7] = bad
        with pytest.raises(BikError, match="outside 0..T"):
            track(lib.bik_track64, q64, tin64, lengths=ln)
    with pytest.raises(BikError, match="T must be at least 1"):
        track(lib.bik_track64, q64, tin64, T=0)
    with pytest.raises(BikError, match="bad argument"):
        conv(lib.bik_converge64, None, inp64)
    with pytest.raises(BikError, match="bad argument"):
        track(lib.bik_track64, None, tin64)
    # nothing was enqueued by the rejected calls: a valid call still runs
    conv(lib.bik_converge64, q64, inp64)
    torch.cuda.synchronize()
