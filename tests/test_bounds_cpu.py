"""Per-instance joint limits (bik_converge_bounded / bik_track_bounded) through the pass loops compiled for the host
(tests/host_emu/emu_bounds.cpp), no GPU needed.

Instance b's bounds narrow the problem's ConfigurationLimit bounds and VelocityLimit caps on the dofs those limits list: bounds
equal to the problem's (or +-inf) give the ..._weighted_ex loops bit for bit, random narrowing gives what a problem built with
the narrowed bounds gives bit for bit, lower == upper == q or a cap of 0 keeps a dof exactly where it is, values on dofs no
limit lists are not read, NaN and inconsistent values are flagged, and bik_track with bounds is one converge per frame.
Cases: g1 and g1_full (a floating base the limits do not list), ur5e_damp, ur5e_wall (collision rows: the general K2) and
TidyBot with a VelocityLimit on its three base joints; every small-group case also on the general path.
"""

import copy

import numpy as np
import pytest

from mink_b200._abi import LIMIT_CONFIGURATION, LIMIT_VELOCITY, LimitSpec
from tests.emu_bounds_lib import PATH_AUTO, PATH_GENERAL, BoundedEmu
from tests.test_posture_weights_cpu import _at, _case, _eq, _lengths

CONV = dict(max_iters=10, pos_threshold=2e-3, ori_threshold=2e-3)
NONFINITE, QP_INFEASIBLE = 4, 8
NAMES = ["g1", "g1_full", "ur5e_damp", "ur5e_wall", "tidybot"]
BASE = [0, 1, 2]   # TidyBot: joint_x, joint_y, joint_th


def _paths(name):
    return [PATH_AUTO] if name == "ur5e_wall" else [PATH_AUTO, PATH_GENERAL]


def _bcase(name, dtype, B, T, seed):
    """tests.test_posture_weights_cpu._case, with TidyBot given a VelocityLimit on its base, and a BoundedEmu on its problem.
    cfg / vel: the problem's per-dof ConfigurationLimit bounds and VelocityLimit caps as the image stores them (fp32), +-inf
    where the limit does not list the dof."""
    c = _case(name, dtype, B, T, seed)
    spec = c["spec"]
    if name == "tidybot":
        spec = copy.deepcopy(spec)
        spec.limits.append(LimitSpec(LIMIT_VELOCITY, dof=np.array(BASE, np.int32), vmax=np.array([0.5, 0.5, 1.0])))
    nv = c["nv"]
    lo, up, vm = np.full(nv, -np.inf), np.full(nv, np.inf), np.full(nv, np.inf)
    for l in spec.limits:
        if l.kind == LIMIT_CONFIGURATION:
            lo[l.dof] = np.float32(l.lower)
            up[l.dof] = np.float32(l.upper)
        elif l.kind == LIMIT_VELOCITY:
            vm[l.dof] = np.minimum(vm[l.dof], np.float32(l.vmax))
    return dict(c, spec=spec, emu=BoundedEmu(c["fm"].to_blob(), spec, c["fm"].nq, nv), cfg=(lo, up), vel=vm)


def _narrowed_spec(spec, lo, up, vm):
    """The problem built with bounds max(lower, lo), min(upper, up) and caps min(vmax, vm) on the dofs each limit lists."""
    s = copy.deepcopy(spec)
    for l in s.limits:
        if l.kind == LIMIT_CONFIGURATION:
            l.lower = np.maximum(np.float32(l.lower).astype(np.float64), lo[l.dof])
            l.upper = np.minimum(np.float32(l.upper).astype(np.float64), up[l.dof])
        elif l.kind == LIMIT_VELOCITY:
            l.vmax = np.minimum(np.float32(l.vmax).astype(np.float64), vm[l.dof])
    return s


def _random_bounds(c, dtype, seed, q0):
    """fp32-representable narrowing per instance: lower / upper inside the problem's range and around q0 (a quarter of them
    with lower == upper), +-inf on a fifth of the dofs, caps in [0, vmax]."""
    rng = np.random.default_rng(seed)
    B, nv, fm = c["B"], c["nv"], c["fm"]
    (lo0, up0), vm0 = c["cfg"], c["vel"]
    qd = np.zeros((B, nv))
    for d in range(nv):
        if fm.dof_qadr[d] >= 0:
            qd[:, d] = q0[:, fm.dof_qadr[d]]
    lo = np.full((B, nv), -np.inf)
    up = np.full((B, nv), np.inf)
    fin = np.isfinite(lo0) & np.isfinite(up0)
    qc = np.clip(qd, lo0, up0)
    with np.errstate(invalid="ignore"):   # (inf - inf on the dofs `fin` leaves out)
        lo[:, fin] = (lo0 + rng.uniform(0, 1, (B, nv)) * (qc - lo0))[:, fin]
        up[:, fin] = (qc + rng.uniform(0, 1, (B, nv)) * (up0 - qc))[:, fin]
    eq = rng.uniform(size=(B, nv)) < 0.25
    up[eq & fin] = lo[eq & fin]
    lo[rng.uniform(size=(B, nv)) < 0.2] = -np.inf
    up[rng.uniform(size=(B, nv)) < 0.2] = np.inf
    vm = np.where(np.isfinite(vm0), rng.uniform(0, 1, (B, nv)) * np.where(np.isfinite(vm0), vm0, 0), np.inf)
    vm[rng.uniform(size=(B, nv)) < 0.1] = 0.0
    vm[rng.uniform(size=(B, nv)) < 0.2] = np.inf
    f32 = lambda a: a.astype(np.float32).astype(dtype)
    has_cfg = np.isfinite(lo0).any() or np.isfinite(up0).any()
    return (f32(lo) if has_cfg else None, f32(up) if has_cfg else None, f32(vm) if np.isfinite(vm0).any() else None)


@pytest.mark.parametrize("dtype", [np.float32, np.float64], ids=["f32", "f64"])
@pytest.mark.parametrize("name", NAMES)
def test_problem_bounds_are_the_identity(name, dtype):
    """Bounds equal to the problem's fp32 values, or +-inf, give the ..._weighted_ex loops bit for bit, with and without
    posture weights, for converge and for track with ragged lengths, on every K2 path of the case."""
    c = _bcase(name, dtype, B=24 + 3, T=3, seed=3)
    B, T, P, nv = c["B"], c["T"], c["P"], c["nv"]
    rng = np.random.default_rng(4)
    (lo0, up0), vm0 = c["cfg"], c["vel"]
    pick = lambda v, inf: np.where(rng.uniform(size=(B, nv)) < 0.3, inf, np.broadcast_to(v, (B, nv))).astype(dtype)
    has_cfg = np.isfinite(lo0).any()
    bd = (pick(lo0, -np.inf) if has_cfg else None, pick(up0, np.inf) if has_cfg else None, pick(vm0, np.inf) if np.isfinite(vm0).any() else None)
    pw = rng.uniform(0.2, 1.0, size=(B, T, P, nv)).astype(dtype) if P else None
    ln = _lengths(B, T, 5)
    for path in _paths(name):
        for w in ([None, pw] if P else [None]):
            w0 = None if w is None else w[:, 0]
            ref = c["emu"].converge(c["q0"], c["ft"][:, 0], c["pt"], _at(c["ct"], 0), None, **c["kw"], **CONV, posture_weights=w0, path=path)
            got = c["emu"].converge(c["q0"], c["ft"][:, 0], c["pt"], _at(c["ct"], 0), bd, **c["kw"], **CONV, posture_weights=w0, path=path)
            for x, y in zip(got, ref):
                _eq(x, y)
            ref = c["emu"].track(c["q0"], c["ft"], c["pt"], c["ct"], None, **c["kw"], **CONV, lengths=ln, posture_weights=w, path=path)
            got = c["emu"].track(c["q0"], c["ft"], c["pt"], c["ct"], bd, **c["kw"], **CONV, lengths=ln, posture_weights=w, path=path)
            for x, y in zip(got, ref):
                _eq(x, y)


@pytest.mark.parametrize("dtype", [np.float32, np.float64], ids=["f32", "f64"])
@pytest.mark.parametrize("name", NAMES)
def test_random_narrowing_is_the_rebuilt_problem(name, dtype):
    """Each instance with random fp32-representable narrowing equals, bit for bit, a problem built with its narrowed bounds:
    q, iterations, status; on every K2 path of the case.  In fp64 one step also matches the fp64 oracle run with those bounds
    (1e-6 rad, the fp64 loops' parity tolerance of tests/test_converge64_cpu.py)."""
    from oracle.ikoracle import Oracle

    c = _bcase(name, dtype, B=10, T=1, seed=21)
    B, nv, fm = c["B"], c["nv"], c["fm"]
    bd = _random_bounds(c, dtype, 22, c["q0"])
    full = [np.full((B, nv), -np.inf) if bd[0] is None else bd[0].astype(np.float64),
            np.full((B, nv), np.inf) if bd[1] is None else bd[1].astype(np.float64),
            np.full((B, nv), np.inf) if bd[2] is None else bd[2].astype(np.float64)]
    ft, ct = c["ft"][:, 0], _at(c["ct"], 0)
    for path in _paths(name):
        q, it, st = c["emu"].converge(c["q0"], ft, c["pt"], ct, bd, **c["kw"], **CONV, path=path)
        q1, _, st1 = c["emu"].converge(c["q0"], ft, c["pt"], ct, bd, **c["kw"], max_iters=1, pos_threshold=0.0, ori_threshold=0.0, path=path)
        for b in range(B):
            spec_b = _narrowed_spec(c["spec"], full[0][b], full[1][b], full[2][b])
            emu_b = BoundedEmu(fm.to_blob(), spec_b, fm.nq, nv)
            sl = slice(b, b + 1)
            pt_b = None if c["pt"] is None else c["pt"][sl]
            qr, itr, str_ = emu_b.converge(c["q0"][sl], ft[sl], pt_b, None if ct is None else ct[sl], None, **c["kw"], **CONV, path=path)
            _eq(q[b], qr[0]); _eq(it[b], itr[0]); _eq(st[b], str_[0])
            if dtype == np.float64 and path == PATH_AUTO and not (st1[b] & ~16):
                orc = Oracle(fm.to_blob(), spec_b, fm.nq, nv)
                f64 = lambda a: None if a is None else np.asarray(a[sl], np.float64)
                _, q_ref, st_ref, _ = orc.step(f64(c["q0"]), f64(ft), f64(c["pt"]), f64(ct), **c["kw"], nsteps=1, integrate=True)
                if not st_ref.any():
                    np.testing.assert_allclose(q1[b], q_ref[0], atol=1e-6, rtol=0)


@pytest.mark.parametrize("dtype", [np.float32, np.float64], ids=["f32", "f64"])
@pytest.mark.parametrize("name", NAMES)
def test_locked_dofs_do_not_move(name, dtype):
    """lower == upper == q0 on a listed dof, or a cap of 0, keeps that dof of that instance exactly at its start through
    converge (even instances: configuration lock; odd ones: cap of 0, where the case has a VelocityLimit)."""
    c = _bcase(name, dtype, B=12, T=1, seed=31)
    B, nv, fm = c["B"], c["nv"], c["fm"]
    (lo0, up0), vm0 = c["cfg"], c["vel"]
    rng = np.random.default_rng(32)
    lo, up, vm = np.full((B, nv), -np.inf, dtype), np.full((B, nv), np.inf, dtype), np.full((B, nv), np.inf, dtype)
    locked = np.zeros((B, nv), bool)
    for b in range(B):
        use_vel = b % 2 == 1 and np.isfinite(vm0).any()
        cand = [d for d in range(nv) if fm.dof_qadr[d] >= 0 and (np.isfinite(vm0[d]) if use_vel else
                (np.isfinite(lo0[d]) and lo0[d] <= c["q0"][b, fm.dof_qadr[d]] <= up0[d]))]
        for d in rng.choice(cand, size=min(3, len(cand)), replace=False):
            locked[b, d] = True
            if use_vel:
                vm[b, d] = 0.0
            else:
                lo[b, d] = up[b, d] = c["q0"][b, fm.dof_qadr[d]]
    has_cfg = np.isfinite(lo0).any()
    bd = (lo if has_cfg else None, up if has_cfg else None, vm if np.isfinite(vm0).any() else None)
    for path in _paths(name):
        q, it, st = c["emu"].converge(c["q0"], c["ft"][:, 0], c["pt"], _at(c["ct"], 0), bd, **c["kw"], **CONV, path=path)
        assert not (st & (NONFINITE | QP_INFEASIBLE)).any(), st
        for b, d in zip(*np.nonzero(locked)):
            a = fm.dof_qadr[d]
            assert q[b, a] == c["q0"][b, a], (path, b, d, q[b, a] - c["q0"][b, a])
        moved = [b for b in range(B) if (q[b] != c["q0"][b]).any()]
        assert moved, "nothing moved: the targets do not exercise the lock"


@pytest.mark.parametrize("dtype", [np.float32, np.float64], ids=["f32", "f64"])
@pytest.mark.parametrize("name", ["g1", "tidybot"])
def test_unlisted_dofs_are_not_read(name, dtype):
    """Values on dofs that no limit lists (G1's floating base, TidyBot's base for the ConfigurationLimit and its arm for the
    base's VelocityLimit) change nothing, bit for bit: finite, inconsistent and NaN alike."""
    c = _bcase(name, dtype, B=16, T=1, seed=41)
    B, nv = c["B"], c["nv"]
    (lo0, up0), vm0 = c["cfg"], c["vel"]
    rng = np.random.default_rng(42)
    unl_cfg = ~(np.isfinite(lo0) | np.isfinite(up0))
    unl_vel = ~np.isfinite(vm0)
    assert unl_cfg.any() or unl_vel.any()
    lo, up, vm = np.full((B, nv), -np.inf, dtype), np.full((B, nv), np.inf, dtype), np.full((B, nv), np.inf, dtype)
    lo[:, unl_cfg] = rng.uniform(0.5, 1.0, (B, int(unl_cfg.sum())))
    up[:, unl_cfg] = -lo[:, unl_cfg]
    up[1::3, unl_cfg] = np.nan
    vm[:, unl_vel] = -rng.uniform(0.0, 1.0, (B, int(unl_vel.sum())))
    vm[2::3, unl_vel] = np.nan
    has_cfg = np.isfinite(lo0).any()
    bd = (lo if has_cfg else None, up if has_cfg else None, vm if np.isfinite(vm0).any() else None)
    for path in _paths(name):
        ref = c["emu"].converge(c["q0"], c["ft"][:, 0], c["pt"], _at(c["ct"], 0), None, **c["kw"], **CONV, path=path)
        got = c["emu"].converge(c["q0"], c["ft"][:, 0], c["pt"], _at(c["ct"], 0), bd, **c["kw"], **CONV, path=path)
        for x, y in zip(got, ref):
            _eq(x, y)


@pytest.mark.parametrize("dtype", [np.float32, np.float64], ids=["f32", "f64"])
@pytest.mark.parametrize("name", ["g1", "ur5e_wall"])
def test_nan_and_inconsistent_bounds_are_flagged(name, dtype):
    """A NaN on a listed dof narrows nothing and sets BIK_STATUS_NONFINITE on that instance only; lower > upper after narrowing,
    or a negative cap, sets BIK_STATUS_QP_INFEASIBLE on that instance only (g1 on the small-group K2, ur5e_wall on the general
    one)."""
    c = _bcase(name, dtype, B=8, T=1, seed=51)
    B, nv, fm = c["B"], c["nv"], c["fm"]
    (lo0, up0), vm0 = c["cfg"], c["vel"]
    d = int(np.nonzero(np.isfinite(lo0) & np.isfinite(vm0))[0][-1])
    lo, up, vm = np.full((B, nv), -np.inf, dtype), np.full((B, nv), np.inf, dtype), np.full((B, nv), np.inf, dtype)
    lo[1, d] = np.nan
    vm[2, d] = np.nan
    lo[4, d], up[4, d] = up0[d], lo0[d]           # lower' = upper_c > upper' = lower_c
    vm[5, d] = -0.5
    args = (c["q0"], c["ft"][:, 0], c["pt"], _at(c["ct"], 0))
    q, it, st = c["emu"].converge(*args, (lo, up, vm), **c["kw"], **CONV)
    q_n, it_n, st_n = c["emu"].converge(*args, None, **c["kw"], **CONV)
    ok = [0, 1, 2, 3, 6, 7]
    _eq(q[ok], q_n[ok]); _eq(it[ok], it_n[ok])
    assert not (st_n & (NONFINITE | QP_INFEASIBLE)).any()
    _eq(st[[0, 3, 6, 7]], st_n[[0, 3, 6, 7]])
    _eq(st[[1, 2]], st_n[[1, 2]] | NONFINITE)
    assert (st[[4, 5]] & QP_INFEASIBLE).all() and not (st[[0, 1, 2, 3, 6, 7]] & QP_INFEASIBLE).any()


@pytest.mark.parametrize("dtype", [np.float32, np.float64], ids=["f32", "f64"])
@pytest.mark.parametrize("name", ["g1", "tidybot", "ur5e_wall"])
@pytest.mark.parametrize("seq", [False, True], ids=["held", "sequence"])
def test_track_equals_per_frame_converge(name, dtype, seq):
    """bik_track_bounded with one row of bounds per instance equals one bounded converge per frame, bit for bit, with ragged
    lengths, per-frame posture weights where the case has posture tasks, and with `sequence` a BIK_POSTURE_SEQ_BATCHED
    posture target sequence."""
    c = _bcase(name, dtype, B=24 + 5, T=3, seed=12)
    B, T, P, nv = c["B"], c["T"], c["P"], c["nv"]
    bd = _random_bounds(c, dtype, 13, c["q0"])
    pw = np.random.default_rng(14).uniform(0.0, 1.0, size=(B, T, P, nv)).astype(dtype) if P else None
    ln = _lengths(B, T, 2)
    pts = (lambda t: c["pseq"][:, t]) if seq else (lambda t: c["pt"])
    q = c["q0"]
    q_loop, it_loop, st_loop = np.zeros((B, T, c["fm"].nq), q.dtype), np.zeros((B, T), np.int32), np.zeros((B, T), np.int32)
    for t in range(T):
        q, it_loop[:, t], st_loop[:, t] = c["emu"].converge(q, c["ft"][:, t], pts(t), _at(c["ct"], t), bd, **c["kw"], **CONV,
                                                            posture_weights=None if pw is None else pw[:, t])
        q_loop[:, t] = q
    q_end, q_traj, it, st, _ = c["emu"].track(c["q0"], c["ft"], c["pseq"] if seq else c["pt"], c["ct"], bd, **c["kw"], **CONV, lengths=ln,
                                              posture_weights=pw, posture_form=3 if seq else None)
    has = np.arange(T)[None, :] < ln[:, None]
    _eq(q_traj[has], q_loop[has])
    _eq(it[has], it_loop[has])
    _eq(st[has], st_loop[has])
    q_ref = np.where(ln[:, None] > 0, q_loop[np.arange(B), np.maximum(ln - 1, 0)], c["q0"])
    _eq(q_end, q_ref)
