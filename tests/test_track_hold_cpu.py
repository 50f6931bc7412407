"""bik_track_hold's pass loop with the kernel headers compiled for the host (tests/host_emu), no GPU needed.

A held task takes, over a run of frames, the value it had at the configuration its run began from.  The emulated
bik_track_hold must equal, bit for bit, the emulated per-frame converge loop in which the caller sets every held task's target
before the first frame of each run from the emulation's own FK at the configuration reached so far (FRAME: world pose,
RELATIVE_FRAME: root^-1 * frame, COM: the CoM, POSTURE: q).  With an all-zero mask it must equal the bik_track_coll loop.
"""

import numpy as np
import pytest

from tests.emu_hold_lib import HoldEmu
from tests.helpers import track_case

CONV = dict(max_iters=10, pos_threshold=2e-3, ori_threshold=2e-3)


def _hemu(name):
    from tests.helpers import load_case
    _, fm, spec, _ = load_case(name)
    return HoldEmu(fm.to_blob(), spec, fm.nq, fm.nv)


def _frame_targets(he, c):
    """[B, T, F, 7] targets of every frame-like task: track_case's sequences for the FRAME tasks, and for a RELATIVE_FRAME task
    its pose in the root at q0 on every frame."""
    from mink_b200._abi import TASK_FRAME, TASK_RELATIVE_FRAME
    cap = he.capture(c["q0"], f64=c["q0"].dtype == np.float64)
    cols, i = [], 0
    for k, t in enumerate([t for t in he.spec.tasks if t.kind in (TASK_FRAME, TASK_RELATIVE_FRAME)]):
        if t.kind == TASK_FRAME:
            cols.append(c["ft"][:, :, i]); i += 1
        else:
            cols.append(np.repeat(cap[k][:, None], c["T"], axis=1))
    return np.ascontiguousarray(np.stack(cols, axis=2))


def _runs(rng, B, T, H):
    """Random run masks: every (instance, task) switches on and off at random frames."""
    hold = rng.random((B, T, H)) < 0.5
    hold[0] = True             # one instance holds everything on every frame
    hold[1] = False
    hold[2, :, :] = np.arange(T)[:, None] % 4 < 2   # runs of two frames
    return hold


def _per_frame_loop(he, c, hold, f64, f32k1):
    """T converge calls; before the first frame of each run, the held task's target is set from FK at the q reached so far."""
    q = c["q0"].copy()
    B, T = c["B"], c["T"]
    ft, ct = _frame_targets(he, c), None if c["ct"] is None else c["ct"].copy()
    pt = np.repeat(c["pt"], he.spec.nposture, axis=1).copy()
    F, Cn = he.spec.nframe, he.spec.ncom
    held = None
    q_traj, it_l, st_l = np.zeros((B, T, q.shape[1]), q.dtype), np.zeros((B, T), np.int32), np.zeros((B, T), np.int32)
    for t in range(T):
        start = hold[:, t] & (~hold[:, t - 1] if t > 0 else True)
        if start.any():
            cap = he.capture(q, f64=f64 or not f32k1)
            held = cap if held is None else [np.where(start[:, k, None], cap[k], held[k]) for k in range(len(cap))]
        ftt, ctt, ptt = ft[:, t].copy(), None if ct is None else ct[:, t].copy(), pt.copy()
        for k in range(hold.shape[2]):
            on = hold[:, t, k]
            if not on.any():
                continue
            if k < F:
                ftt[on, k] = held[k][on]
            elif k < F + Cn:
                ctt[on, k - F] = held[k][on]
            else:
                ptt[on, k - F - Cn] = held[k][on]
        q, it_l[:, t], st_l[:, t] = he.converge(q, ftt, ptt, ctt, **c["kw"], **CONV, f32k1=f32k1)
        q_traj[:, t] = q
    return q_traj, it_l, st_l


@pytest.mark.parametrize("name", ["edge", "g1"])
@pytest.mark.parametrize("dtype", [np.float32, np.float64])
def test_emulated_hold_equals_per_frame_loop(name, dtype):
    """edge: every task kind (FRAME, RELATIVE_FRAME, COM, POSTURE), a collision limit and a floating root; g1: the headline
    humanoid.  fp32 runs K1 in fp32 (BIK_K1_PRECISION=f32), so the emulated fp32 bik_fk is the reference."""
    he = _hemu(name)
    c = track_case(name, B=37, T=9, seed=5, dtype=dtype)
    f64 = dtype == np.float64
    H = he.spec.nframe + he.spec.ncom + he.spec.nposture
    hold = _runs(np.random.default_rng(3), c["B"], c["T"], H)
    pt = np.repeat(c["pt"], he.spec.nposture, axis=1)
    q_end, q_traj, it, st, _ = he.track_hold(c["q0"], _frame_targets(he, c), pt, c["ct"], hold, **c["kw"], **CONV, f32k1=not f64)
    q_ref, it_ref, st_ref = _per_frame_loop(he, c, hold, f64, f32k1=not f64)
    np.testing.assert_array_equal(it, it_ref)
    np.testing.assert_array_equal(st, st_ref)
    np.testing.assert_array_equal(q_traj, q_ref)
    np.testing.assert_array_equal(q_end, q_ref[:, -1])
    # everything held on every frame: the instance stays where it is, one step per frame
    assert (it[0] == 1).all()
    tol = 1e-12 if f64 else 1e-6
    np.testing.assert_allclose(q_traj[0], np.repeat(c["q0"][:1], c["T"], axis=0), atol=tol, rtol=0)


@pytest.mark.parametrize("name", ["edge", "g1"])
@pytest.mark.parametrize("dtype", [np.float32, np.float64])
def test_emulated_zero_mask_equals_track_coll(name, dtype):
    """An all-zero mask runs the hold instantiation of K1 and K2 on ptcur, and gives what bik_track_coll gives, bit for bit."""
    he = _hemu(name)
    c = track_case(name, B=29, T=6, seed=9, dtype=dtype)
    H = he.spec.nframe + he.spec.ncom + he.spec.nposture
    pt = np.repeat(c["pt"], he.spec.nposture, axis=1)
    ln = np.random.default_rng(1).integers(0, c["T"] + 1, size=c["B"]).astype(np.int32)
    zero = np.zeros((c["B"], c["T"], H), bool)
    ft = _frame_targets(he, c)
    a = he.track_hold(c["q0"], ft, pt, c["ct"], zero, **c["kw"], **CONV, lengths=ln)
    b = he.track_hold(c["q0"], ft, pt, c["ct"], None, **c["kw"], **CONV, lengths=ln)
    for x, y in zip(a, b):
        np.testing.assert_array_equal(x, y)
