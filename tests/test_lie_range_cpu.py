"""The Lie layer of K1 (mink_b200/csrc/bik_math.h) over the whole rotation range, fp32 and fp64, against tests/lie_ref.

bik_math.h has four regimes: the identity branch of the SE(3) inverse left Jacobian (|w|^2 < 1e-10), the Maclaurin series
of its coefficients below theta^2 = 1, their closed forms above, and the log's branch flip at theta = pi.  Frame targets
drawn by perturbing joints stay below ~0.7 rad, so these tests place targets at prescribed angles (helpers.LIE_ANGLES)
instead, and compare with an extended-precision reference rather than with the C oracle: the oracle's closed form for the
SO(3) inverse left Jacobian cancels below theta ~ 1e-2 (test_oracle_small_angle_band pins how much).  Everything runs on the
kernel headers compiled for the host (tests/host_emu); tests/test_gpu_lie_range.py runs the same cases on the device.
"""

import functools

import numpy as np
import pytest

from tests import lie_ref
from tests.emu_lib import Emu, lie_coefs, lie_quat_integrate, lie_quat_sub
from tests.helpers import (LIE_ANGLES, LIE_CASES, LIE_OFFSETS, chain_case, lie_case, lie_targets, lie_task_rows, load_case,
                           make_inputs, qmul_np, targets_at_angle, task_frames)

EPS = np.finfo(np.float64).eps
IDENTITY_STRADDLE = LIE_ANGLES[2:4]   # 1e-5 (1 -/+ 1e-3)
B = 12
# fp64 kernel ("f64", and "mixed": the fp64 kernel on fp32 inputs): absolute on e and J.  fp32 kernel: 3-5x the largest
# deviation the host emulation shows over the grid (FK in fp32 included).
BARS = {"f64": (1e-13, 1e-13), "mixed": (1e-13, 1e-13), "f32": (2e-6, 4e-6)}
# ball64's tip sits behind 62 joints, whose fp32 FK rounding the Lie layer inherits: 2.0e-6 on e and 2.8e-6 on J on the host
F32_BARS_LONG_CHAIN = (6e-6, 1e-5)
# coefficient functions, relative.  fp64: everywhere (the closed-form D loses most just above theta = 1, 2.5e-14).  fp32:
# twice the largest the host shows over the grid, 1.5e-5, which is D's closed form just above theta = 1, where
# 2 th - 3 sin th + th cos th cancels to ~th^5 / 60 (A 1.1e-6, C 1.8e-6, B 2.8e-7 there); the series below it are good to ~1 ulp
COEF_BAR = {True: 5e-14, False: 3e-5}


def _r32(a):
    return None if a is None else np.asarray(a, np.float32).astype(np.float64)


@functools.lru_cache(maxsize=None)
def _case(cid):
    c = lie_case(cid)
    c["emu"] = Emu(c["fm"].to_blob(), c["spec"], c["fm"].nq, c["fm"].nv)
    inp = make_inputs(c["fm"], c["wl"], B, c["fk"], seed=3, sigma=0.3)
    c["q"], c["pt"] = inp["q"], inp["posture_target"]
    return c


@functools.lru_cache(maxsize=None)
def _grid_inputs(cid, r32):
    """[(theta, offset, q, ft, pt, e_ref, J_ref)] over LIE_ANGLES x LIE_OFFSETS; inputs rounded to fp32 when r32, and the
    reference evaluated on exactly those inputs."""
    c = _case(cid)
    rng = np.random.default_rng(11)
    out = []
    for theta in LIE_ANGLES:
        for off in LIE_OFFSETS:
            q, pt = c["q"], c["pt"]
            ft = lie_targets(c, q, theta, off, rng)
            if r32:
                q, ft, pt = _r32(q), _r32(ft), _r32(pt)
            e, J = lie_task_rows(c, q, ft)
            out.append((theta, off, q, ft, pt, e, J))
    return out


# ---- coefficient functions ------------------------------------------------------------------------------------------------
def _t2_grid():
    return np.unique(np.concatenate([
        [0.0], np.logspace(-20, -1, 400), 1e-10 * (1 + np.linspace(-1e-2, 1e-2, 41)),    # around the identity switch
        np.linspace(0, np.pi ** 2, 4001), 1 + np.linspace(-1e-3, 1e-3, 81), 1 + np.logspace(-15, -3, 60),   # the series switch
        1 - np.logspace(-15, -3, 60), np.pi ** 2 - np.logspace(-12, 0, 40)]))


@pytest.mark.parametrize("f64", [True, False], ids=["f64", "f32"])
def test_coefficients_against_mpmath(f64):
    """coef_A / coef_BCD on a dense theta^2 grid over [0, pi^2], packed around 1e-10 and 1: relative error of A, B, C, D."""
    t2 = _t2_grid()
    if not f64:
        t2 = np.unique(_r32(t2))
    got, ref = lie_coefs(t2, f64), lie_ref.coefs(t2)
    rel = np.abs(got - ref) / np.abs(ref)
    worst = rel.max(0)
    where = t2[rel.argmax(0)]
    print(f"{'f64' if f64 else 'f32'}: max rel err A {worst[0]:.1e} (t2={where[0]:.6g}) B {worst[1]:.1e} (t2={where[1]:.6g}) "
          f"C {worst[2]:.1e} (t2={where[2]:.6g}) D {worst[3]:.1e} (t2={where[3]:.6g})")
    assert worst.max() <= COEF_BAR[f64], (worst, where)


# ---- K1 over the angle grid -----------------------------------------------------------------------------------------------
@pytest.mark.parametrize("prec", ["f64", "mixed", "f32"])
@pytest.mark.parametrize("cid", list(LIE_CASES))
def test_k1_frame_rows_against_mpmath(cid, prec):
    """Emu.fk_jac's frame-task rows (e, J) at every angle and offset of the grid against the extended-precision reference
    on the same inputs: fp64 inputs for "f64", fp32-rounded ones for "f32" and "mixed"."""
    c = _case(cid)
    te, tJ = F32_BARS_LONG_CHAIN if (prec == "f32" and cid == "ball64") else BARS[prec]
    worst_e = worst_J = 0.0
    for theta, off, q, ft, pt, e_ref, J_ref in _grid_inputs(cid, prec != "f64"):
        J, e, *_ = c["emu"].fk_jac(q, ft, pt, prec=prec)
        if prec == "f32" and theta in IDENTITY_STRADDLE:
            # fp32 FK rounds |w| by ~1e-7 rad, 1 % of it here: which side of the switch J lands on is the kernel's e's call
            _, J_ref = lie_task_rows(c, q, ft, e_like=e.astype(np.float64))
        de = np.abs(e[:, :e_ref.shape[1]] - e_ref).max()
        dJ = np.abs(J[:, :J_ref.shape[1]] - J_ref).max()
        worst_e, worst_J = max(worst_e, de), max(worst_J, dJ)
        assert de <= te and dJ <= tJ, (theta, off, de, dJ)
    print(f"{cid}/{prec}: max|e - e_ref| {worst_e:.1e} max|J - J_ref| {worst_J:.1e}")


@pytest.mark.parametrize("prec", ["f64", "f32"])
@pytest.mark.parametrize("cid", ["n7", "rel7"])
def test_k1_at_exactly_pi_and_target_sign(cid, prec):
    """At theta = pi (target rotation with w = 0 exactly) either sign of the rotation is a log: the kernel's is +-the
    reference's with |w| = pi, v is the reference's on that side, and J is the reference J at the kernel's own e.  Then on the whole grid: negating the target quaternions gives bit-identical
    e and J."""
    c = _case(cid)
    r32 = prec == "f32"
    te, tJ = BARS[prec]
    rng = np.random.default_rng(5)
    for off in LIE_OFFSETS:
        ft = lie_targets(c, c["q"], np.pi, off, rng)
        q, ft, pt = (_r32(a) for a in (c["q"], ft, c["pt"])) if r32 else (c["q"], ft, c["pt"])
        J, e, *_ = c["emu"].fk_jac(q, ft, pt, prec=prec)
        e_pos, _ = lie_task_rows(c, q, ft)
        e = e[:, :e_pos.shape[1]].astype(np.float64)
        e_ref, J_ref = lie_task_rows(c, q, ft, e_like=e)
        for k in range(e_ref.shape[1] // 6):   # the rotation is +-the reference's, |w| = pi
            w, w_pos = e[:, 6 * k + 3:6 * k + 6], e_pos[:, 6 * k + 3:6 * k + 6]
            assert np.minimum(np.abs(w - w_pos).max(1), np.abs(w + w_pos).max(1)).max() <= te, (off, k)
            assert np.abs(np.linalg.norm(w, axis=1) - np.pi).max() <= te, (off, k)
        assert np.abs(e - e_ref).max() <= te, (off, np.abs(e - e_ref).max())
        assert np.abs(J[:, :J_ref.shape[1]] - J_ref).max() <= tJ, (off, np.abs(J[:, :J_ref.shape[1]] - J_ref).max())
    for theta, off, q, ft, pt, _, _ in _grid_inputs(cid, r32):
        neg = ft.copy()
        neg[..., :4] *= -1
        a = c["emu"].fk_jac(q, ft, pt, prec=prec)
        b = c["emu"].fk_jac(q, neg, pt, prec=prec)
        assert np.array_equal(a[0], b[0]) and np.array_equal(a[1], b[1]), (theta, off)


# ---- ball-joint posture rows and integration ------------------------------------------------------------------------------
POSTURE_ANGLES = (0.0, 1e-9, 1e-4, 0.5, 1.0, 2.0, 3.0, np.pi - 1e-3, np.pi + 1e-3, 4.0, 5.5, 2 * np.pi - 1e-3)


def _rotated(qb, theta, rng):
    """qb * exp(theta * a) for random unit axes a, in the hemisphere the product lands in (w < 0 past pi)."""
    ax = rng.normal(size=(len(qb), 3))
    ax /= np.linalg.norm(ax, axis=1, keepdims=True)
    return qmul_np(qb, np.concatenate([np.full((len(qb), 1), np.cos(theta / 2)), np.sin(theta / 2) * ax], 1))


@pytest.mark.parametrize("f64", [True, False], ids=["f64", "f32"])
def test_quat_sub_past_pi_both_hemispheres(f64):
    """quat_sub (the ball-joint posture error, mju_subQuat) at angles up to and past pi, with the target in either
    hemisphere (q and -q): past pi the angle wraps to (-pi, pi].  Then the same error as ep, K1's posture rows, on the
    ball64 chain."""
    rng = np.random.default_rng(21)
    tol = 1e-14 if f64 else 2e-6
    qb = rng.normal(size=(64, 4))
    qb /= np.linalg.norm(qb, axis=1, keepdims=True)
    for theta in POSTURE_ANGLES:
        qa = _rotated(qb, theta, rng)
        for sgn in (1.0, -1.0):
            a, b = (qa * sgn, qb) if f64 else (_r32(qa * sgn), _r32(qb))
            got, ref = lie_quat_sub(a, b, f64), lie_ref.quat_sub(a, b)
            assert np.abs(got - ref).max() <= tol, (theta, sgn, np.abs(got - ref).max())
            assert np.all(np.linalg.norm(ref, axis=1) <= np.pi + 1e-12)
    c = _case("ball64")
    fm = c["fm"]
    n = [i for i in range(fm.nnode) if int(fm.node_type[i]) == 1][0]   # the ball joint
    qa_, da = int(fm.node_qadr[n]), int(fm.node_dadr[n])
    prec = "f64" if f64 else "f32"
    for theta in POSTURE_ANGLES:
        q = c["q"].copy()
        pt = np.tile(c["pt"], (B, 1))
        pt[:, qa_:qa_ + 4] = _rotated(q[:, qa_:qa_ + 4], theta, rng) * rng.choice([-1.0, 1.0], size=(B, 1))
        if not f64:
            q, pt = _r32(q), _r32(pt)
        ft = lie_targets(c, q, 0.3, 0.1, rng)
        _, _, ep, *_ = c["emu"].fk_jac(q, ft, pt, prec=prec)
        ref = lie_ref.quat_sub(pt[:, qa_:qa_ + 4], q[:, qa_:qa_ + 4])
        assert np.abs(ep[:, 0, da:da + 3] - ref).max() <= tol, theta


INTEGRATE_NORMS = (0.0, 1e-16, 1e-8, 1.0, np.pi, 2 * np.pi - 1e-3, 5.0)


@pytest.mark.parametrize("f64", [True, False], ids=["f64", "f32"])
@pytest.mark.parametrize("cid", ["free32", "ball64"])
def test_integrate_free_and_ball_joints(cid, f64):
    """integrate_instance with rotation steps |w| in INTEGRATE_NORMS on the free / ball joint: the quaternion against
    quat_integrate in extended precision, the other coordinates against q + dq; then quat_integrate alone."""
    c = _case(cid)
    fm = c["fm"]
    rng = np.random.default_rng(31)
    kind = 0 if cid == "free32" else 1
    n = [i for i in range(fm.nnode) if int(fm.node_type[i]) == kind][0]
    qa, da = int(fm.node_qadr[n]) + (3 if kind == 0 else 0), int(fm.node_dadr[n]) + (3 if kind == 0 else 0)
    tol = 1e-15 if f64 else 4e-7
    for norm in INTEGRATE_NORMS:
        dq = rng.normal(0, 0.05, size=(B, fm.nv))
        ax = rng.normal(size=(B, 3))
        dq[:, da:da + 3] = norm * ax / np.linalg.norm(ax, axis=1, keepdims=True)
        q = c["q"]
        if not f64:
            q, dq = _r32(q), _r32(dq)
        got = c["emu"].integrate(q, dq, f64=f64).astype(np.float64)
        ref_q = lie_ref.quat_integrate(q[:, qa:qa + 4], dq[:, da:da + 3])
        assert np.abs(got[:, qa:qa + 4] - ref_q).max() <= tol, (norm, np.abs(got[:, qa:qa + 4] - ref_q).max())
        rest = np.ones(fm.nq, bool)
        rest[qa:qa + 4] = False
        lin = q + 0.0
        for d in range(fm.nv):
            if int(fm.dof_qadr[d]) >= 0:
                lin[:, int(fm.dof_qadr[d])] += dq[:, d]
        if kind == 0:
            lin[:, qa - 3:qa] += dq[:, da - 3:da]
        assert np.abs(got[:, rest] - lin[:, rest]).max() <= (1e-15 if f64 else 4e-7) * 4, norm
        assert np.abs(lie_quat_integrate(q[:, qa:qa + 4], dq[:, da:da + 3], f64) - ref_q).max() <= tol, norm


# ---- why the reference is not the oracle below 1e-2 rad -------------------------------------------------------------------
def test_oracle_small_angle_band():
    """The C oracle's so3_ljacinv uses the reference's cancelling closed form from theta = 1e-5 up; its J deviates from the
    extended-precision one by about 2 eps / theta^2 there.  Pinned under 4 eps / theta^2 across 1e-5 < theta < 1e-2, and
    above the fp64 bars of this file at 1e-4, which is why those compare with tests/lie_ref and not with the oracle."""
    c = _case("n7")
    rng = np.random.default_rng(41)
    dev = {}
    for theta in np.logspace(np.log10(1.2e-5), -2, 13):
        ft = lie_targets(c, c["q"], theta, 0.3, rng)
        Jo, eo, _ = c["orc"].fk_jac(c["q"], ft, c["pt"])
        e, J = lie_task_rows(c, c["q"], ft)
        dev[theta] = np.abs(Jo[:, :6] - J).max()
        assert np.abs(eo[:, :6] - e).max() <= 1e-14
        assert dev[theta] <= 4 * EPS / theta ** 2, (theta, dev[theta])
    print("oracle J deviation: " + ", ".join(f"{t:.1e}: {d:.1e}" for t, d in dev.items()))
    t = min(dev, key=lambda x: abs(np.log(x / 1e-4)))
    assert dev[t] > BARS["f64"][1]


# ---- the converge loop from far-away targets ------------------------------------------------------------------------------
FAR_ANGLES = (2.5, 3.0, np.pi - 1e-2)
CONV = dict(max_iters=12, pos_threshold=2e-3, ori_threshold=2e-3)


def _far_case(name):
    if name == "ur5e":
        wl, fm, spec, _ = load_case("ur5e")
        from oracle.ikoracle import Oracle
        orc = Oracle(fm.to_blob(), spec, fm.nq, fm.nv)
        frames = task_frames(wl, fm)
        c = dict(fm=fm, wl=wl, spec=spec, orc=orc, frames=frames, fk=lambda qq: orc.fk(qq, frames))
        c["emu"] = Emu(fm.to_blob(), spec, fm.nq, fm.nv)
        inp = make_inputs(fm, wl, 3 * B, c["fk"], seed=8, sigma=0.3)
        c["q"], c["pt"] = inp["q"], inp["posture_target"]
        return c
    c = chain_case(7, seed=7)
    c["emu"] = Emu(c["fm"].to_blob(), c["spec"], c["fm"].nq, c["fm"].nv)
    inp = make_inputs(c["fm"], c["wl"], 3 * B, c["fk"], seed=8, sigma=0.3)
    c["q"], c["pt"] = inp["q"], inp["posture_target"]
    return c


@functools.lru_cache(maxsize=None)
def far_converge_inputs(name):
    """(case, q0, targets) with each instance's target 2.5 .. pi - 1e-2 rad from its frame (0.05 m away), and the oracle's
    converge loop on them in fp64 and on their fp32 rounding."""
    c = _far_case(name)
    rng = np.random.default_rng(51)
    poses, _ = c["orc"].fk(c["q"], c["frames"], want_com=False)
    n = len(c["q"]) // len(FAR_ANGLES)
    ft = np.concatenate([targets_at_angle(poses[k * n:(k + 1) * n, 0], th, 0.05, rng) for k, th in enumerate(FAR_ANGLES)])[:, None]
    kw = dict(dt=c["wl"]["dt"], damping=c["wl"]["damping"])
    ref64 = c["orc"].converge(c["q"], ft, c["pt"], None, **kw, **CONV)
    ref32 = c["orc"].converge(_r32(c["q"]), _r32(ft), _r32(c["pt"]), None, **kw, **CONV)
    return c, ft, kw, ref64, ref32


@pytest.mark.parametrize("name", ["n7", "ur5e"])
def test_converge_from_far_targets(name):
    """Emu.converge (the pass loop of bik_converge64 / bik_converge) against Oracle.converge: fp64 with the same iteration
    counts and flags and q within 1e-6; fp32 with the same flags and q within 1e-3 (tests/test_track_cpu.py's bar)."""
    c, ft, kw, ref64, ref32 = far_converge_inputs(name)
    q, it, st = c["emu"].converge(c["q"], ft, c["pt"], None, **kw, **CONV)
    assert int((st & 15).max()) == 0
    np.testing.assert_array_equal(it, ref64[1])
    np.testing.assert_array_equal((st & 16) == 0, ref64[2].astype(bool))
    d64 = np.abs(q - ref64[0]).max()
    assert d64 <= 1e-6, d64   # tests/test_converge64_cpu.py's bar; 4.8e-7 on ur5e here, 1.1e-7 on n7
    q32, it32, st32 = c["emu"].converge(c["q"].astype(np.float32), ft.astype(np.float32), c["pt"].astype(np.float32), None, **kw, **CONV)
    assert int((st32 & 15).max()) == 0
    np.testing.assert_array_equal((st32 & 16) == 0, ref32[2].astype(bool))
    d32 = np.abs(q32 - ref32[0]).max()
    print(f"{name}: converged {int(ref64[2].sum())}/{len(it)}, iters {np.bincount(it).tolist()}, fp64 max|dq| {d64:.1e}, "
          f"fp32 {d32:.1e} ({int((it32 != ref32[1]).sum())} iteration counts differ)")
    assert d32 <= 1e-3, d32
