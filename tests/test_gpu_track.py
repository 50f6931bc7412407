"""bik_track / Problem.track / track_ik: the converge loop over a sequence of targets, every instance on its own frame cursor.

The contract: for every instance b, bik_track gives bit for bit what T calls of bik_converge give, one per frame on the same
buffers -- only without the per-frame barrier between instances.  Targets come from the C oracle's FK along a seeded, smooth
joint path q0 (+) (t+1)/T delta.
"""

import os

import numpy as np
import pytest

torch = pytest.importorskip("torch")
pytestmark = pytest.mark.gpu

from mink_b200.workloads import make_inputs  # noqa: E402
from tests.helpers import load_case, task_frames  # noqa: E402


def _need_gpu():
    if not torch.cuda.is_available():
        pytest.skip("no CUDA device")


def _case(name, B, T, seed, sigma=0.3):
    _need_gpu()
    from mink_b200.engine import DeviceModel, Problem
    from oracle.ikoracle import Oracle

    wl, fm, spec, g = load_case(name)
    model = DeviceModel(fm, device=0)
    prob = Problem(model, spec)
    orc = Oracle(fm.to_blob(), spec, fm.nq, fm.nv)
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
    dev = lambda a: None if a is None else torch.tensor(np.ascontiguousarray(a), dtype=torch.float32, device="cuda:0")
    ft = dev(np.asarray(poses).reshape(B, T, -1, 7))
    ct = dev(np.asarray(com).reshape(B, T, -1, 3)) if spec.ncom else None
    pt = dev(inp["q"][:, None, :])   # each instance's posture target is its start: the frame tasks can be met
    kw = dict(dt=wl["dt"], damping=wl["damping"])
    return dict(wl=wl, fm=fm, spec=spec, prob=prob, orc=orc, q0=inp["q"], ft=ft, ct=ct, pt=pt, kw=kw, B=B, T=T)


def _q(c):
    return torch.tensor(c["q0"], dtype=torch.float32, device="cuda:0")


def _per_frame(c, **kw):
    """The contract's loop: one Problem.converge call per frame on the same q."""
    q = _q(c)
    qs, its, sts = [], [], []
    for t in range(c["T"]):
        it, st = c["prob"].converge(q, c["ft"][:, t], c["pt"], None if c["ct"] is None else c["ct"][:, t], **c["kw"], **kw)
        qs.append(q.clone()); its.append(it.clone()); sts.append(st.clone())
    return torch.stack(qs, 1), torch.stack(its, 1), torch.stack(sts, 1), q


def _track(c, lengths=None, **kw):
    q = _q(c)
    q_traj, it, st, passes = c["prob"].track(q, c["ft"], c["pt"], c["ct"], lengths=lengths, **c["kw"], **kw)
    return q_traj, it, st, q, int(passes)


class _graph_mode:
    def __init__(self, mode):
        self.mode = mode

    def __enter__(self):
        os.environ["BIK_CONVERGE_GRAPH"] = self.mode

    def __exit__(self, *a):
        os.environ.pop("BIK_CONVERGE_GRAPH", None)


def _equal(a, b):
    assert torch.equal(a.cpu(), b.cpu()), f"{int((a.cpu() != b.cpu()).sum())} elements differ"


CONV = dict(max_iters=10, pos_threshold=2e-3, ori_threshold=2e-3)


@pytest.mark.parametrize("mode", ["1", "0"])
@pytest.mark.parametrize("name", ["ur5e", "g1", "h1", "ur5e_wall"])
def test_track_equals_the_per_frame_converge_loop(name, mode):
    """ur5e: small-group K2; g1: fp32 K1, velocity box; h1: CoM trajectory; ur5e_wall: collision rows (fp64 K1, general K2).
    Graph mode ("1") and the host-polled loop ("0", polled every 3 passes)."""
    c = _case(name, B=1000 + 13, T=12, seed=21)
    with _graph_mode(mode):
        q_loop, it_loop, st_loop, q_end = _per_frame(c, check_every=3, **CONV)
        q_traj, it, st, q, passes = _track(c, check_every=3, **CONV)
    _equal(q_traj, q_loop)
    _equal(it, it_loop)
    _equal(st, st_loop)
    _equal(q, q_end)
    its = it.cpu().numpy().astype(np.int64) + 1
    print(f"{name}: iters histogram {np.bincount(its.ravel() - 1).tolist()} passes {passes} "
          f"per-frame barrier {int(its.max(0).sum())}")
    # no per-frame barrier: each instance runs its own sum of passes, the batch the longest of them
    assert passes == int(its.sum(1).max())
    if name == "ur5e":   # (the humanoids miss the thresholds on most frames: there the slowest instance is the same one)
        assert passes < int(its.max(0).sum())


def test_track_lengths():
    """Mixed lengths, 0 and T included: each instance matches the loop over its own frames; rows past its length keep the
    NaN / -1 sentinel; q ends at the end of its last frame."""
    c = _case("ur5e", B=500 + 7, T=9, seed=33)
    B, T = c["B"], c["T"]
    ln = np.random.default_rng(3).integers(0, T + 1, size=B).astype(np.int32)
    ln[:3] = [0, T, 1]
    q_loop, it_loop, st_loop, _ = _per_frame(c, **CONV)
    q_traj, it, st, q, passes = _track(c, lengths=torch.tensor(ln, device="cuda:0"), **CONV)
    q_loop, it_loop, st_loop = q_loop.cpu().numpy(), it_loop.cpu().numpy(), st_loop.cpu().numpy()
    q_traj, it, st, q = q_traj.cpu().numpy(), it.cpu().numpy(), st.cpu().numpy(), q.cpu().numpy()
    has = np.arange(T)[None, :] < ln[:, None]
    np.testing.assert_array_equal(q_traj[has], q_loop[has])
    np.testing.assert_array_equal(it[has], it_loop[has])
    np.testing.assert_array_equal(st[has], st_loop[has])
    assert np.isnan(q_traj[~has]).all() and (it[~has] == -1).all() and (st[~has] == -1).all()
    q_ref = np.where(ln[:, None] > 0, q_loop[np.arange(B), np.maximum(ln - 1, 0)], c["q0"].astype(np.float32))
    np.testing.assert_array_equal(q, q_ref)
    assert passes == int(np.where(has, it + 1, 0).sum(1).max())


def test_track_rejects_bad_lengths():
    from mink_b200._lib import BikError

    c = _case("ur5e", B=16, T=4, seed=1)
    for bad in (-1, 5):
        ln = torch.full((16,), 2, dtype=torch.int32, device="cuda:0")
        ln[7] = bad
        with pytest.raises(BikError, match="outside 0..T"):
            _track(c, lengths=ln, **CONV)


def test_track_against_oracle():
    """The oracle's converge loop in fp64, frame after frame: iteration counts agree on >= 99.5 % of (b, t); where an
    instance's counts agree up to frame t, q_traj[b][t] is within 1e-3 (the bar of test_converge_batch_against_oracle)."""
    c = _case("ur5e", B=1000 + 13, T=12, seed=44)
    q_traj, it, st, _, _ = _track(c, **CONV)
    q_traj, it = q_traj.cpu().numpy(), it.cpu().numpy()
    ft, pt = c["ft"].cpu().numpy().astype(np.float64), c["pt"].cpu().numpy().astype(np.float64)
    q = c["q0"].astype(np.float32).astype(np.float64)
    q_ref, it_ref = np.zeros_like(q_traj, dtype=np.float64), np.zeros_like(it)
    for t in range(c["T"]):
        q, it_ref[:, t], _, _ = c["orc"].converge(q, ft[:, t], pt, None, **c["kw"], **CONV)
        q_ref[:, t] = q
    same = it == it_ref
    print(f"track vs oracle: mismatching iters {int((~same).sum())}/{same.size}")
    assert same.mean() >= 0.995
    upto = np.cumprod(same, axis=1).astype(bool)
    np.testing.assert_allclose(q_traj[upto], q_ref[upto], atol=1e-3)


def test_track_graph_cache():
    """Two identical calls give identical results (the cached graph is replayed); a track -> converge -> track sequence on one
    problem gives the standalone results (the cache key includes the mode)."""
    c = _case("ur5e", B=300 + 5, T=6, seed=55)
    a = _track(c, **CONV)
    b = _track(c, **CONV)
    for x, y in zip(a[:4], b[:4]):
        _equal(x, y)
    assert a[4] == b[4]
    q = _q(c)
    it_alone, st_alone = c["prob"].converge(q, c["ft"][:, 0], c["pt"], None, **c["kw"], **CONV)
    q_alone = q.clone()
    _track(c, **CONV)
    q = _q(c)
    it2, st2 = c["prob"].converge(q, c["ft"][:, 0], c["pt"], None, **c["kw"], **CONV)
    _equal(it2, it_alone)
    _equal(st2, st_alone)
    _equal(q, q_alone)
    d = _track(c, **CONV)
    for x, y in zip(a[:4], d[:4]):
        _equal(x, y)


def _g1_api(B, T, seed=7):
    import mink_b200 as mink
    from mink_b200.lie import SE3

    c = _case("g1", B=B, T=T, seed=seed)
    wl, fm = c["wl"], c["fm"]

    def setup(q0, posture):
        cfg = mink.Configuration(fm, q0)
        tasks = [mink.FrameTask(f["name"], f["type"], f["position_cost"], f["orientation_cost"], lm_damping=f["lm_damping"])
                 for f in wl["frames"]]
        post = mink.PostureTask(fm, cost=wl["posture"]["cost"])
        post.set_target(posture)
        limits = [mink.ConfigurationLimit(fm),
                  mink.VelocityLimit(fm, {n: np.pi for n, t in zip(fm.names["joint"], fm.node_type) if t >= 2})]
        pelvis = cfg.get_transform_frame_to_world(wl["frames"][2]["name"], wl["frames"][2]["type"])
        tasks[2].set_target(pelvis)   # held for every frame
        return cfg, tasks + [post], limits

    return c, setup, mink, SE3


def test_track_ik_equals_converge_ik_frame_by_frame():
    """G1: foot FrameTask sequences, a held pelvis target and a PostureTask.  track_ik on a batch == converge_ik after
    set_target on every frame; a single Configuration gets numpy back and ends at its final q."""
    c, setup, mink, SE3 = _g1_api(B=96, T=6)
    ft = c["ft"].cpu().numpy().astype(np.float64)
    dt, damping = c["kw"]["dt"], c["kw"]["damping"]
    conv = dict(max_iters=10, pos_threshold=2e-3, ori_threshold=2e-3)
    q0 = torch.tensor(c["q0"], dtype=torch.float32, device="cuda:0")

    pt = c["pt"][:, 0].cpu().numpy().astype(np.float64)
    cfg, tasks, limits = setup(q0.clone(), pt)
    feet = {tasks[0]: c["ft"][:, :, 0], tasks[1]: SE3(ft[:, :, 1])}   # a CUDA tensor and an SE3
    q_traj, iters, ok = mink.track_ik(cfg, tasks, dt, feet, damping=damping, limits=limits, **conv)
    assert isinstance(q_traj, torch.Tensor) and q_traj.shape == (96, 6, c["fm"].nq) and ok.dtype == torch.bool

    cfg2, tasks2, limits2 = setup(q0.clone(), pt)
    for t in range(6):
        tasks2[0].set_target(SE3(ft[:, t, 0]))
        tasks2[1].set_target(SE3(ft[:, t, 1]))
        it, okt = mink.converge_ik(cfg2, tasks2, dt, damping=damping, limits=limits2, **conv)
        _equal(q_traj[:, t], cfg2.q_device)
        np.testing.assert_array_equal(iters[:, t].cpu().numpy(), it)
        np.testing.assert_array_equal(ok[:, t].cpu().numpy(), okt)
    _equal(cfg.q_device, cfg2.q_device)

    # one configuration: numpy out, shared [T, 7] sequences, the configuration ends at its last frame
    one, tasks1, limits1 = setup(c["q0"][0], pt[0])
    q1, it1, ok1 = mink.track_ik(one, tasks1, dt, {tasks1[0]: ft[0, :, 0], tasks1[1]: ft[0, :, 1]}, damping=damping,
                                 limits=limits1, **conv)
    assert isinstance(q1, np.ndarray) and q1.shape == (6, c["fm"].nq) and it1.shape == (6,) and ok1.dtype == bool
    np.testing.assert_array_equal(one.q, q1[-1])


def test_track_ik_errors():
    c, setup, mink, SE3 = _g1_api(B=8, T=3)
    ft = c["ft"].cpu().numpy().astype(np.float64)
    dt = c["kw"]["dt"]
    cfg, tasks, limits = setup(torch.tensor(c["q0"], dtype=torch.float32, device="cuda:0"), c["pt"][:, 0].cpu().numpy())
    with pytest.raises(mink.TargetNotSet):   # the right foot has neither a sequence nor a target
        mink.track_ik(cfg, tasks, dt, {tasks[0]: ft[:, :, 0]}, limits=limits)
    with pytest.raises(mink.InvalidTarget):   # not [T, 7] / [B, T, 7]
        mink.track_ik(cfg, tasks, dt, {tasks[0]: ft[:, :, 0, :6], tasks[1]: ft[:, :, 1]}, limits=limits)
    with pytest.raises(mink.InvalidTarget):   # sequences of different lengths
        mink.track_ik(cfg, tasks, dt, {tasks[0]: ft[:, :, 0], tasks[1]: ft[:, :2, 1]}, limits=limits)
    with pytest.raises(mink.InvalidTarget):   # lengths for another batch size
        mink.track_ik(cfg, tasks, dt, {tasks[0]: ft[:, :, 0], tasks[1]: ft[:, :, 1]}, limits=limits, lengths=np.ones(5, np.int32))
