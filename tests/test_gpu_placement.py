"""Per-instance frame placement on the device: bik_step_placed / bik_converge_placed / bik_track_placed (and their fp64 forms)
through Problem.step / converge / track, and the `placement=` mapping of converge_ik.

NULL placement and rows equal to the problem's own placement give the ..._coll / bik_track_hold entry points bit for bit;
a few thousand instances over eight placements give, group by group, the problems built with them bit for bit; fp64 agrees
with the C oracle run per placement; a UR5e tool-length sweep through converge_ik equals, instance for instance, converge_ik
on models whose attachment_site was moved, and every placed TCP ends on its target.  Then the cached converge graph
following the placement buffer, and the C ABI's refusals.
"""

import ctypes as C
import os

import numpy as np
import pytest

torch = pytest.importorskip("torch")
pytestmark = pytest.mark.gpu

from tests.emu_placement_lib import own_placement, placed_spec  # noqa: E402
from tests.test_gpu_posture_weights import _problem  # noqa: E402
from tests.test_placement_cpu import CONV, NAMES, _case as _ccase, _placements  # noqa: E402
from tests.test_posture_weights_cpu import _lengths  # noqa: E402
from tests.test_track_hold_cpu import _runs  # noqa: E402

DT = {np.float32: torch.float32, np.float64: torch.float64}
F32K1 = {"BIK_K1_PRECISION": "f32"}


def _case(name, dtype, B, T, seed, env=None):
    if not torch.cuda.is_available():
        pytest.skip("no CUDA device")
    c = _ccase(name, dtype, B=B, T=T, seed=seed)
    c["env"] = env
    c["prob"] = _problem(c["fm"], c["spec"], env)
    c["dev"] = lambda a, dt=DT[dtype]: None if a is None else torch.tensor(np.ascontiguousarray(a), dtype=dt, device="cuda:0")
    c["d"] = {k: c["dev"](c[k]) for k in ("ft", "ct", "pt")}
    return c


class _Null:
    """A placement whose pointer is NULL: Problem.step / converge / track then call the ..._placed entry points with NULL."""

    def data_ptr(self):
        return 0


def _call(c, mode, placement, prob=None, sl=slice(None), hold=None, lengths=None, null=False):
    """The call `mode` (step, converge, track) on instances `sl`; returns its outputs as a tuple of tensors."""
    prob = prob or c["prob"]
    d, dev = c["d"], c["dev"]
    q = dev(c["q0"][sl])
    ct = None if d["ct"] is None else d["ct"][sl]
    pl = None if placement is None else dev(placement)
    if null:
        prob._placement = lambda *a: _Null()
    try:
        if mode == "step":
            dq, st = prob.step(q, d["ft"][sl, 0], d["pt"][sl], None if ct is None else ct[:, 0], nsteps=3, integrate=True, placement=pl, **c["kw"])
            return q, dq, st
        if mode == "converge":
            it, st = prob.converge(q, d["ft"][sl, -1], d["pt"][sl], None if ct is None else ct[:, -1], placement=pl, **c["kw"], **CONV)
            return q, it, st
        h = None if hold is None else dev(np.asarray(hold[sl], np.uint8), torch.uint8)
        ln = None if lengths is None else dev(lengths[sl], torch.int32)
        out = prob.track(q, d["ft"][sl], d["pt"][sl], ct, lengths=ln, hold=h, placement=pl, **c["kw"], **CONV)
        return (q,) + tuple(out)
    finally:
        if null:
            del prob._placement


def _equal(a, b):
    for x, y in zip(a, b):
        torch.testing.assert_close(x, y, rtol=0, atol=0, equal_nan=True)


@pytest.mark.parametrize("dtype", [np.float32, np.float64], ids=["f32", "f64"])
@pytest.mark.parametrize("name", NAMES)
def test_null_and_own_placement_are_the_entry_points_without_one(name, dtype):
    """NULL placement runs what bik_step_coll / bik_converge_coll / bik_track_hold run; rows equal to the problem's own
    placement give the same bit for bit where K1 runs in the inputs' precision (fp64, or fp32 with BIK_K1_PRECISION=f32)."""
    for env in ([None, F32K1] if dtype == np.float32 else [None]):
        c = _case(name, dtype, B=200 + 3, T=3, seed=3, env=env)
        B, T = c["B"], c["T"]
        own = own_placement(c["spec"], B, dtype)
        hold = _runs(np.random.default_rng(4), B, T, c["spec"].nframe + c["spec"].ncom + c["spec"].nposture)
        ln = _lengths(B, T, 5)
        for mode, kw in (("step", {}), ("converge", {}), ("track", dict(lengths=ln)), ("track", dict(lengths=ln, hold=hold))):
            ref = _call(c, mode, None, **kw)
            _equal(_call(c, mode, own, null=True, **kw), ref)
            if dtype == np.float64 or env is not None:
                _equal(_call(c, mode, own, **kw), ref)


@pytest.mark.parametrize("dtype", [np.float32, np.float64], ids=["f32", "f64"])
@pytest.mark.parametrize("name", NAMES)
def test_per_instance_placements_are_the_rebuilt_problems(name, dtype):
    """3 000 instances over eight placements (unit quaternions with components in {0, +-0.5, +-1}, positions exact in fp32):
    every group equals the problem built with its placement, bit for bit (dq, q, q_traj, iters, status)."""
    c = _case(name, dtype, B=3000, T=3, seed=11)
    B, K = c["B"], 8
    pls = _placements(np.random.default_rng(12), c["spec"], K, dtype, own_first=False)
    group = np.random.default_rng(13).integers(0, K, size=B)
    rows = pls[group]
    hold = _runs(np.random.default_rng(14), B, c["T"], c["spec"].nframe + c["spec"].ncom + c["spec"].nposture)
    ln = _lengths(B, c["T"], 15)
    for mode, kw in (("step", {}), ("converge", {}), ("track", dict(lengths=ln, hold=hold))):
        out = _call(c, mode, rows, **kw)
        for g in range(K):
            idx = np.nonzero(group == g)[0]
            ref = _call(c, mode, None, prob=_problem(c["fm"], placed_spec(c["spec"], pls[g])), sl=idx, **kw)
            for x, y in zip(out[:4], ref[:4]):   # (track's passes count the whole batch: not compared)
                torch.testing.assert_close(x[torch.as_tensor(idx, device=x.device)], y, rtol=0, atol=0, equal_nan=True)


# device fp64 against the C oracle after three integrated steps: UR5e agrees to 1e-9 rad; the G1 and edge QPs are less well
# conditioned (up to 1.6e-8 rad in the host emulation of the kernels), and the problem without a placement is held to the same bar
ORACLE_TOL = {"ur5e": 1e-9, "g1": 5e-8, "edge": 5e-8}


def _oracle_placements(rng, spec, K):
    """[K, F, 7] fp64 placements for the oracle comparison: each frame turned by 0.2 rad about a random axis and moved by up to
    0.1 in its node.  (Half-turn placements, as _placements draws, put the frame errors near pi, where the device and the
    oracle may take different branches of the logarithm; the rebuilt-problem tests cover those bit for bit.)"""
    from tests.helpers import qmul_np

    own = own_placement(spec, 1, np.float64)[0]
    out = np.repeat(own[None], K, axis=0)
    for k in range(K):
        for f in range(own.shape[0]):
            ax = rng.normal(size=3)
            ax /= np.linalg.norm(ax)
            out[k, f, :4] = qmul_np(own[f, :4], np.concatenate([[np.cos(0.1)], np.sin(0.1) * ax]))
            out[k, f, 4:] += rng.uniform(-0.1, 0.1, size=3)
    return out


@pytest.mark.parametrize("name", NAMES)
def test_fp64_against_the_oracle_per_placement(name):
    """bik_step_placed64 (three integrated steps) against oracle/ik_oracle.c run on the problem of each placement, within
    the device's agreement with the oracle (ORACLE_TOL), which the problem without a placement meets as well."""
    from oracle.ikoracle import Oracle

    c = _case(name, np.float64, B=64, T=1, seed=21)
    K = 4
    pls = _oracle_placements(np.random.default_rng(22), c["spec"], K)
    group = np.arange(c["B"]) % K
    q, _, _ = _call(c, "step", pls[group])
    q = q.cpu().numpy()
    fm = c["fm"]
    for g in range(K):
        idx = np.nonzero(group == g)[0]
        orc = Oracle(fm.to_blob(), placed_spec(c["spec"], pls[g]), fm.nq, fm.nv)
        ct = None if c["ct"] is None else c["ct"][idx, 0]
        _, q_ref, _, _ = orc.step(c["q0"][idx], c["ft"][idx, 0], c["pt"][idx], ct, **c["kw"], nsteps=3, integrate=True)
        np.testing.assert_allclose(q[idx], q_ref, rtol=0, atol=ORACLE_TOL[name])
    q, _, _ = _call(c, "step", None)
    ct = None if c["ct"] is None else c["ct"][:, 0]
    _, q_ref, _, _ = Oracle(fm.to_blob(), c["spec"], fm.nq, fm.nv).step(c["q0"], c["ft"][:, 0], c["pt"], ct, **c["kw"], nsteps=3, integrate=True)
    np.testing.assert_allclose(q.cpu().numpy(), q_ref, rtol=0, atol=ORACLE_TOL[name])


def test_tool_length_sweep_through_converge_ik(tmp_path):
    """A UR5e whose attachment_site sits at one of eight tool lengths per instance: converge_ik(placement=) equals, instance
    for instance and bit for bit in fp64, converge_ik on a model whose site_pos holds that tool's pose, and every placed TCP
    ends within the thresholds of its target."""
    if not torch.cuda.is_available():
        pytest.skip("no CUDA device")
    import mink_b200 as mink
    from mink_b200.lie import SE3
    from tests.helpers import extract_example_scenes

    path = os.path.join(extract_example_scenes(str(tmp_path)), "universal_robots_ur5e", "scene.xml")
    model = mink.Model.from_xml_path(path)
    sid = mink.flatten(model).names["site"].index("attachment_site")
    p0, q0 = np.array(model.site_pos[sid], dtype=np.float64), np.array(model.site_quat[sid], dtype=np.float64)
    lengths = np.arange(8) * 0.025   # tool lengths along the site's z axis
    w, x, y, z = q0 / np.linalg.norm(q0)
    axis = np.array([2 * (x * z + w * y), 2 * (y * z - w * x), 1 - 2 * (x * x + y * y)])
    tools = np.array([np.concatenate([q0, p0 + L * axis]) for L in lengths])
    B = 8 * 40
    tool = np.arange(B) % 8
    rng = np.random.default_rng(31)
    flat = mink.flatten(model)
    home = flat.key("home") if "home" in flat.names["key"] else np.asarray(flat.qpos0, dtype=np.float64)
    q_start = home + rng.normal(0.0, 0.3, size=(B, model.nq))
    q_goal = q_start + rng.normal(0.0, 0.15, size=(B, model.nq))

    def moved(k):
        m = mink.Model.from_xml_path(path)
        m.site_pos[sid], m.site_quat[sid] = tools[k, 4:], tools[k, :4]
        return m

    # targets: the placed TCP at q_goal, from the moved model's FK
    targets = np.zeros((B, 7))
    for k in range(8):
        idx = np.nonzero(tool == k)[0]
        targets[idx] = mink.Configuration(moved(k), torch.tensor(q_goal[idx])).get_transform_frame_to_world("attachment_site", "site").wxyz_xyz

    def solve(m, q, tgt, placement=None):
        cfg = mink.Configuration(m, torch.tensor(q))
        tcp = mink.FrameTask("attachment_site", "site", position_cost=1.0, orientation_cost=1.0)
        tcp.set_target(SE3(tgt))
        it, ok = mink.converge_ik(cfg, [tcp], 0.01, damping=1e-3, limits=[mink.ConfigurationLimit(m)], max_iters=200,
                                  pos_threshold=1e-4, ori_threshold=1e-4, placement=None if placement is None else {tcp: placement})
        return cfg.q, it, ok

    q, it, ok = solve(model, q_start, targets, torch.tensor(tools[tool]))
    for k in range(8):
        idx = np.nonzero(tool == k)[0]
        m = moved(k)
        q_ref, it_ref, ok_ref = solve(m, q_start[idx], targets[idx])
        torch.testing.assert_close(q[torch.as_tensor(idx, device=q.device)], q_ref, rtol=0, atol=0)
        np.testing.assert_array_equal(it[idx], it_ref)
        np.testing.assert_array_equal(ok[idx], ok_ref)
        pose = mink.Configuration(m, q_ref).get_transform_frame_to_world("attachment_site", "site")
        err = SE3(targets[idx]).inverse() @ pose
        assert ok[idx].all()
        assert np.linalg.norm(err.translation(), axis=-1).max() <= 2e-4
    # the sweep is a sweep: a longer tool (instance 1) ends elsewhere than the model's own site would for the same target
    assert not torch.equal(q[1], solve(model, q_start[1:2], targets[1:2])[0][0])


def test_graph_cache_follows_the_placement_buffer():
    """Two converge calls that differ only in the placement buffer give their own results (the cached graph is keyed on it)."""
    c = _case("g1", np.float32, B=256, T=1, seed=41, env=F32K1)
    pls = _placements(np.random.default_rng(42), c["spec"], 2, np.float32, own_first=False)
    a, b = (np.ascontiguousarray(np.broadcast_to(p, (c["B"],) + p.shape)) for p in pls)
    r1 = _call(c, "converge", a)
    r2 = _call(c, "converge", b)
    r3 = _call(c, "converge", a)
    _equal(r3, r1)
    assert not torch.equal(r1[0], r2[0])
    _equal(r2, _call(c, "converge", b, prob=_problem(c["fm"], c["spec"], F32K1)))   # a problem without a cached graph


def test_refusals():
    """BIK_ERR_INVALID for a placement on a problem without frame tasks, and for fp64 inputs on an fp32 entry point."""
    if not torch.cuda.is_available():
        pytest.skip("no CUDA device")
    from mink_b200._abi import TASK_POSTURE, BikInputs, ProblemSpec, TaskSpec

    c = _case("ur5e", np.float32, B=4, T=1, seed=51)
    fm, B = c["fm"], c["B"]
    lib = c["prob"].lib
    q = c["dev"](c["q0"])
    pl = c["dev"](own_placement(c["spec"], B, np.float32))
    dq = torch.empty((B, fm.nv), device="cuda:0")
    st = torch.empty(B, device="cuda:0", dtype=torch.int32)
    it = torch.empty(B, device="cuda:0", dtype=torch.int32)
    posture_only = _problem(fm, ProblemSpec([TaskSpec(TASK_POSTURE, dof_cost=np.ones(fm.nv))], []))
    inp = BikInputs()
    inp.posture_targets = c["d"]["pt"].data_ptr()
    inp.posture_batched = 1
    assert lib.bik_converge_placed(posture_only.handle, B, q.data_ptr(), C.byref(inp), None, None, None, None, pl.data_ptr(), 0.01, 1e-3, 5,
                                   1e-3, 1e-3, 1, it.data_ptr(), st.data_ptr(), None) == -1
    assert lib.bik_step_placed(posture_only.handle, B, q.data_ptr(), C.byref(inp), None, None, None, None, pl.data_ptr(), 0.01, 1e-3, 1, 0,
                               dq.data_ptr(), st.data_ptr(), None) == -1
    assert lib.bik_step_placed(posture_only.handle, B, q.data_ptr(), C.byref(inp), None, None, None, None, None, 0.01, 1e-3, 1, 0,
                               dq.data_ptr(), st.data_ptr(), None) == 0   # NULL: the call without a placement
    inp, keep, _, _ = c["prob"]._inputs(None, c["d"]["ft"][:, 0].double(), c["d"]["pt"].double(), None, dtype=torch.float64)
    assert lib.bik_step_placed(c["prob"].handle, B, q.data_ptr(), C.byref(inp), None, None, None, None, pl.data_ptr(), 0.01, 1e-3, 1, 0,
                               dq.data_ptr(), st.data_ptr(), None) == -1
    with pytest.raises(ValueError):
        c["prob"].step(q, c["d"]["ft"][:, 0], c["d"]["pt"], None, placement=pl[:, :, :6])
