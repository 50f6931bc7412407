"""Per-instance frame placement with the kernel headers compiled for the host (tests/host_emu), no GPU needed.

bik_step_placed, bik_converge_placed and bik_track_placed give each instance its own pose of every frame task's frame in its
tree node.  The emulated calls must give each instance, bit for bit, what the same emulated call gives on a problem built
with that instance's placement, for rows that hold exactly what that problem's image holds; rows equal to the problem's own
placement must give the calls without a placement; a non-finite row falls back to the problem's placement and flags the
instance.  Then the front end: the `placement=` mapping's refusals, and its composed rows against flatten on a model whose
site_pos / site_quat were set to the same pose.
"""

import os

import numpy as np
import pytest

from tests.emu_hold_lib import HoldEmu
from tests.emu_placement_lib import PlacementEmu, frame_tasks, image_row, own_placement, placed_spec
from tests.helpers import load_case, track_case
from tests.test_track_hold_cpu import _frame_targets, _runs

CONV = dict(max_iters=10, pos_threshold=2e-3, ori_threshold=2e-3)
NAMES = ["ur5e", "g1", "edge"]
NONFINITE = 4
# unit quaternions with components in {0, +-0.5, +-1}: the builder's normalisation leaves them as they are in fp32 and fp64
QUATS = np.array([[1, 0, 0, 0], [0, 1, 0, 0], [0, 0, 0, -1], [0.5, 0.5, 0.5, 0.5], [0.5, -0.5, 0.5, -0.5], [-0.5, 0.5, 0.5, -0.5]])


def _case(name, dtype, B, T, seed):
    _, fm, spec, _ = load_case(name)
    c = track_case(name, B=B, T=T, seed=seed, dtype=dtype)
    c["fm"], c["spec"] = fm, spec
    c["ft"] = _frame_targets(HoldEmu(fm.to_blob(), spec, fm.nq, fm.nv), c)   # a RELATIVE_FRAME task's target: its pose at q0
    c["pt"] = np.repeat(c["pt"], spec.nposture, axis=1)
    return c


def _placements(rng, spec, K, dtype, own_first=True):
    """[K, F, 7] distinct placements: group 0 the problem's own (own_first), the others unit quaternions of QUATS and positions
    that are multiples of 1/64 within 0.125 of the problem's frame origin (exact in fp32)."""
    own = own_placement(spec, 1, dtype)[0]
    out = [own] if own_first else []
    while len(out) < K:
        rows = own.copy()
        for f in range(own.shape[0]):
            rows[f, :4] = QUATS[rng.integers(len(QUATS))]
            rows[f, 4:] = np.round(np.asarray(frame_tasks(spec)[f].frame.pos) * 64) / 64 + rng.integers(-8, 9, 3) / 64
        out.append(rows.astype(dtype))
    return np.stack(out)


def _run(emu, c, mode, sl, placement, hold=None, lengths=None):
    """The call `mode` (step, converge, track) on instances `sl` of the case."""
    q0, ft, pt, ct = c["q0"][sl], c["ft"][sl], c["pt"][sl], None if c["ct"] is None else c["ct"][sl]
    f32k1 = c["q0"].dtype == np.float32
    if mode == "step":
        return emu.step(q0, ft[:, 0], pt, None if ct is None else ct[:, 0], placement, **c["kw"], nsteps=3, f32k1=f32k1)
    if mode == "converge":
        return emu.converge(q0, ft[:, -1], pt, None if ct is None else ct[:, -1], placement, **c["kw"], **CONV, f32k1=f32k1)
    return emu.track(q0, ft, pt, ct, placement, **c["kw"], **CONV, hold=None if hold is None else hold[sl],
                     lengths=None if lengths is None else lengths[sl], f32k1=f32k1)


def _emu(c, spec=None):
    fm = c["fm"]
    return PlacementEmu(fm.to_blob(), spec or c["spec"], fm.nq, fm.nv)


def _equal(a, b):
    for x, y in zip(a, b):
        np.testing.assert_array_equal(x, y)


MODES = ["step", "converge", "track", "track_hold"]


@pytest.mark.parametrize("mode", MODES)
@pytest.mark.parametrize("dtype", [np.float32, np.float64], ids=["f32", "f64"])
@pytest.mark.parametrize("name", NAMES)
def test_each_instance_is_the_problem_built_with_its_placement(name, dtype, mode):
    """Four placements over 24 instances: every group equals, bit for bit, the same emulated call on a problem built with its
    placement (dq, q, q_traj, iters, status, passes).  fp32 callers run K1 in fp32, where the rows are the image's values."""
    c = _case(name, dtype, B=24, T=4, seed=31)
    B, K = c["B"], 4
    rng = np.random.default_rng(32)
    pls = _placements(rng, c["spec"], K, dtype)
    group = np.arange(B) % K
    rows = np.ascontiguousarray(pls[group])
    hold = None
    if mode == "track_hold":
        hold = _runs(np.random.default_rng(33), B, c["T"], c["spec"].nframe + c["spec"].ncom + c["spec"].nposture)
    mode = mode.replace("_hold", "")
    ln = np.random.default_rng(34).integers(1, c["T"] + 1, size=B).astype(np.int32) if mode == "track" else None
    out = _run(_emu(c), c, mode, slice(None), rows, hold, ln)
    for g in range(K):
        idx = np.nonzero(group == g)[0]
        ref = _run(_emu(c, placed_spec(c["spec"], pls[g])), c, mode, idx, None, hold, ln)
        for x, y in zip(out, ref):
            if np.ndim(x) == 0:
                continue   # passes: a count of the whole batch
            np.testing.assert_array_equal(np.asarray(x)[idx], y)
    # the placements moved the solution: a group other than the problem's own ends elsewhere
    assert not np.array_equal(out[0][group == 1], _run(_emu(c), c, mode, np.nonzero(group == 1)[0], None, hold, ln)[0])


@pytest.mark.parametrize("mode", MODES)
@pytest.mark.parametrize("dtype", [np.float32, np.float64], ids=["f32", "f64"])
@pytest.mark.parametrize("name", NAMES)
def test_own_placement_is_the_call_without_one(name, dtype, mode):
    """Rows equal to the problem's own placement give the ..._coll / bik_track_hold emulation's outputs bit for bit."""
    c = _case(name, dtype, B=13, T=3, seed=41)
    hold = None
    if mode == "track_hold":
        hold = _runs(np.random.default_rng(42), c["B"], c["T"], c["spec"].nframe + c["spec"].ncom + c["spec"].nposture)
    mode = mode.replace("_hold", "")
    emu = _emu(c)
    _equal(_run(emu, c, mode, slice(None), own_placement(c["spec"], c["B"], dtype), hold), _run(emu, c, mode, slice(None), None, hold))


@pytest.mark.parametrize("mode", ["step", "converge", "track"])
@pytest.mark.parametrize("dtype", [np.float32, np.float64], ids=["f32", "f64"])
@pytest.mark.parametrize("name", ["g1", "edge"])
def test_nonfinite_row_falls_back_and_flags(name, dtype, mode):
    """A NaN or inf in a row: that task keeps the problem's placement for that instance, which gets BIK_STATUS_NONFINITE (in
    track on every frame it runs); the other instances are untouched."""
    c = _case(name, dtype, B=9, T=3, seed=51)
    rows = own_placement(c["spec"], c["B"], dtype).copy()
    rows[2, 0, 5] = np.nan
    rows[5, -1, 0] = np.inf
    emu = _emu(c)
    out, ref = _run(emu, c, mode, slice(None), rows), _run(emu, c, mode, slice(None), None)
    st, st_ref = out[-2] if mode == "track" else out[-1], ref[-2] if mode == "track" else ref[-1]
    for k, (x, y) in enumerate(zip(out, ref)):
        if x is st:
            continue
        np.testing.assert_array_equal(x, y)
    bad = np.zeros(c["B"], bool)
    bad[[2, 5]] = True
    ran = st_ref >= 0
    np.testing.assert_array_equal(np.where(ran, st, 0), np.where(ran, st_ref | np.where(bad, NONFINITE, 0).reshape((-1,) + (1,) * (st.ndim - 1)), 0))
    assert ((st[bad] & NONFINITE) != 0)[ran[bad]].all()


# ---------------------------------------------------------------- front end ----------------------------------------------
def _ur5e(examples_dir):
    import mink_b200 as mink

    return mink.Model.from_xml_path(os.path.join(examples_dir, "universal_robots_ur5e", "scene.xml"))


@pytest.fixture(scope="module")
def examples(tmp_path_factory):
    from tests.helpers import extract_example_scenes

    return extract_example_scenes(str(tmp_path_factory.mktemp("examples")))


def _q(B, dtype, nq):
    import torch

    return torch.zeros((B, nq), dtype=dtype)


def test_placement_mapping_refusals(examples):
    import torch

    import mink_b200 as mink
    from mink_b200.exceptions import InvalidTarget
    from mink_b200.ik import _placement

    model = _ur5e(examples)
    flat = mink.flatten(model)
    tcp = mink.FrameTask("attachment_site", "site", position_cost=1.0, orientation_cost=1.0)
    post = mink.PostureTask(model, cost=1e-3)
    other = mink.FrameTask("wrist_3_link", "body", position_cost=1.0, orientation_cost=1.0)
    q = _q(4, torch.float32, flat.nq)
    pose = [1, 0, 0, 0, 0, 0, 0.1]
    assert _placement([tcp, post], None, q, flat) is None
    with pytest.raises(InvalidTarget):
        _placement([tcp, post], {post: pose}, q, flat)            # not a frame task
    with pytest.raises(InvalidTarget):
        _placement([tcp, post], {other: pose}, q, flat)           # not in the task list
    for bad in ([1, 0, 0, 0, 0, 0], np.zeros((3, 7)), np.zeros((4, 2, 7))):
        with pytest.raises(InvalidTarget):
            _placement([tcp, post], {tcp: bad}, q, flat)          # wrong shapes
    old = flat.site_bodyid
    flat.site_bodyid = None                                        # a model whose metadata does not record site bodies
    try:
        with pytest.raises(InvalidTarget):
            _placement([tcp], {tcp: pose}, q, flat)
    finally:
        flat.site_bodyid = old


@pytest.mark.parametrize("dtype", ["float32", "float64"])
def test_composed_rows_are_flatten_of_the_moved_site(examples, dtype):
    """The rows `placement=` hands the device equal, bit for bit, what the problem image of a model whose site_pos /
    site_quat (geom_pos / geom_quat) hold the pose would hold; tasks left out keep the model's, a body frame placed at
    identity is the body itself."""
    import torch

    import mink_b200 as mink
    from mink_b200.ik import _placement
    from mink_b200.lie import SE3

    tdt = getattr(torch, dtype)
    model = _ur5e(examples)
    flat = mink.flatten(model)
    sid = flat.names["site"].index("attachment_site")
    gname = next(n for n in flat.names["geom"] if n)
    gid = flat.names["geom"].index(gname)
    tcp = mink.FrameTask("attachment_site", "site", position_cost=1.0, orientation_cost=1.0)
    geo = mink.FrameTask(gname, "geom", position_cost=1.0, orientation_cost=1.0)
    body = mink.FrameTask("wrist_2_link", "body", position_cost=1.0, orientation_cost=1.0)
    kept = mink.FrameTask("wrist_3_link", "body", position_cost=1.0, orientation_cost=1.0)
    tasks = [tcp, geo, body, kept]
    rng = np.random.default_rng(7)
    B = 5
    poses = np.concatenate([rng.normal(size=(B, 4)), rng.normal(scale=0.1, size=(B, 3))], axis=1)
    poses[3] = poses[1]   # repeated poses share one composition
    gpose = np.concatenate([[0.9, 0.1, -0.2, 0.3], [0.01, -0.02, 0.03]])
    rows = _placement(tasks, {tcp: torch.tensor(poses), geo: SE3(gpose), body: [1, 0, 0, 0, 0, 0, 0]}, _q(B, tdt, flat.nq), flat)
    assert rows.dtype == tdt and tuple(rows.shape) == (B, 4, 7)
    rows = rows.numpy()
    for b in range(B):
        m = _ur5e(examples)
        m.site_pos[sid], m.site_quat[sid] = poses[b, 4:], poses[b, :4]
        m.geom_pos[gid], m.geom_quat[gid] = gpose[4:], gpose[:4]
        fm = mink.flatten(m)
        np.testing.assert_array_equal(rows[b, 0], image_row(fm.site_frames[sid], dtype))
        np.testing.assert_array_equal(rows[b, 1], image_row(fm.geom_frames[gid], dtype))
    bf = flat.frame("wrist_2_link", "body")
    np.testing.assert_allclose(rows[:, 2], np.broadcast_to(image_row(bf, dtype), (B, 7)), rtol=0, atol=1e-15 if dtype == "float64" else 1e-7)
    np.testing.assert_array_equal(rows[:, 3], np.broadcast_to(image_row(flat.frame("wrist_3_link", "body"), dtype), (B, 7)))


def test_site_bodyid_round_trips_the_metadata(examples):
    import mink_b200 as mink

    fm = mink.flatten(_ur5e(examples))
    assert fm.site_bodyid is not None and len(fm.site_bodyid) == len(fm.names["site"])
    back = mink.FlatModel.from_blob(fm.to_blob(), fm.to_meta_json())
    np.testing.assert_array_equal(back.site_bodyid, fm.site_bodyid)
    assert load_case("ur5e")[1].site_bodyid is None   # metadata written before site bodies were recorded still loads
