"""K1's Lie layer over the whole rotation range on the device, against the extended-precision reference (tests/lie_ref).

The cases of tests/test_lie_range_cpu.py, through the CUDA kernels: there sincosf, atan2f and the rsqrt-plus-Newton inv_sqrt
replace glibc's functions.  One ragged batch (B = 3 * 64 + 37) per case carries every (angle, offset) pair of the grid
(helpers.LIE_ANGLES x LIE_OFFSETS), instance b taking pair b mod 45.  fk_jac, the packed K1 form of step / step64, converge /
converge64 and integrate / integrate64 are checked.
"""

import contextlib
import functools
import os

import numpy as np
import pytest

torch = pytest.importorskip("torch")
pytestmark = pytest.mark.gpu

from tests import lie_ref  # noqa: E402
from tests.helpers import (LIE_ANGLES, LIE_CASES, LIE_OFFSETS, chain_case, lie_case, lie_targets, lie_task_rows, load_case,  # noqa: E402
                           make_inputs, targets_at_angle, task_frames)

B = 3 * 64 + 37
PAIRS = [(t, o) for t in LIE_ANGLES for o in LIE_OFFSETS]
IDENTITY_STRADDLE = LIE_ANGLES[2:4]
# tests/test_lie_range_cpu.py's bars: fp64 kernel absolute on e and J; fp32 kernel 3-5x the host emulation's deviation
BARS = {torch.float64: (1e-13, 1e-13), torch.float32: (2e-6, 4e-6)}
# ball64: the fp32 FK rounding of 62 joints (host: 2.0e-6 on e, 2.8e-6 on J; an H100: 3.1e-6 on e at theta = 3, 3.9e-6
# on J at theta = pi - 1e-2)
F32_BARS_LONG_CHAIN = (6e-6, 1e-5)


def _need_gpu():
    if not torch.cuda.is_available():
        pytest.skip("no CUDA device")


@contextlib.contextmanager
def _env(env):
    old = {k: os.environ.get(k) for k in env}
    os.environ.update({k: str(v) for k, v in env.items()})
    try:
        yield
    finally:
        for k, v in old.items():
            if v is None:
                os.environ.pop(k, None)
            else:
                os.environ[k] = v


def _np(t):
    return t.detach().cpu().numpy().astype(np.float64)


def _r32(a):
    return np.asarray(a, np.float32).astype(np.float64)


def _t(a, dtype):
    return torch.tensor(np.ascontiguousarray(a), dtype=dtype, device="cuda:0")


# ---- cases, problems, inputs --------------------------------------------------------------------------------------------
@functools.lru_cache(maxsize=None)
def _case(cid):
    from mink_b200.engine import DeviceModel

    _need_gpu()
    c = lie_case(cid)
    c["model"] = DeviceModel(c["fm"], device=0)
    inp = make_inputs(c["fm"], c["wl"], B, c["fk"], seed=3, sigma=0.3)
    c["q"], c["pt"] = inp["q"], inp["posture_target"]
    return c


def _problem(cid, env=None):
    from mink_b200.engine import Problem

    c = _case(cid)
    with _env(env or {}):
        return Problem(c["model"], c["spec"])


def _grid_targets(c, q, rng):
    """Frame targets [B, F, 7]: instance b at PAIRS[b % len(PAIRS)] from its frames' poses at q."""
    ft = np.zeros((len(q), len(c["frames"]) + (1 if "rel_frames" in c else 0), 7))
    for k, (theta, off) in enumerate(PAIRS):
        idx = np.arange(k, len(q), len(PAIRS))
        ft[idx] = lie_targets(c, q[idx], theta, off, rng)
    return ft


@functools.lru_cache(maxsize=None)
def _inputs(cid):
    """(q, ft, pt) in fp64 and rounded to fp32, with the reference rows on each."""
    c = _case(cid)
    ft = _grid_targets(c, c["q"], np.random.default_rng(11))
    in64 = (c["q"], ft, c["pt"])
    in32 = tuple(_r32(a) for a in in64)
    return dict(in64=in64, in32=in32, ref64=lie_task_rows(c, *in64[:2]), ref32=lie_task_rows(c, *in32[:2]))


def _straddle():
    """Instances whose angle sits next to the identity switch."""
    return np.array([PAIRS[b % len(PAIRS)][0] in IDENTITY_STRADDLE for b in range(B)])


# ---- fk_jac -------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("dtype", [torch.float64, torch.float32], ids=["f64", "f32"])
@pytest.mark.parametrize("cid", list(LIE_CASES))
def test_fk_jac_against_mpmath(cid, dtype):
    """bik_fk_jac[64]'s frame-task rows at every (angle, offset) against the reference on the same inputs; for fp32, at
    the angles that straddle the identity switch J is compared at the kernel's own e (fp32 FK's rounding decides the side)."""
    c = _case(cid)
    inp = _inputs(cid)
    f64 = dtype == torch.float64
    q, ft, pt = inp["in64"] if f64 else inp["in32"]
    e_ref, J_ref = inp["ref64"] if f64 else inp["ref32"]
    J, e, *_ = _problem(cid).fk_jac(_t(q, dtype), _t(ft, dtype), _t(pt, dtype), None, dt=c["wl"]["dt"])
    n = e_ref.shape[1]
    J, e = _np(J)[:, :n], _np(e)[:, :n]
    if not f64:
        s = _straddle()
        J_ref = J_ref.copy()
        J_ref[s] = lie_task_rows(c, q[s], ft[s], e_like=e[s])[1]
    te, tJ = F32_BARS_LONG_CHAIN if (not f64 and cid == "ball64") else BARS[dtype]
    de, dJ = np.abs(e - e_ref).max(1), np.abs(J - J_ref).max((1, 2))
    worst = lambda d: f"{d.max():.1e} at theta={PAIRS[int(d.argmax()) % len(PAIRS)][0]:.6g} offset={PAIRS[int(d.argmax()) % len(PAIRS)][1]:g}"
    print(f"{cid}/{'f64' if f64 else 'f32'}: max|e - e_ref| {worst(de)}, max|J - J_ref| {worst(dJ)}")
    assert de.max() <= te and dJ.max() <= tJ


@pytest.mark.parametrize("dtype", [torch.float64, torch.float32], ids=["f64", "f32"])
@pytest.mark.parametrize("cid", ["n7", "rel7"])
def test_fk_jac_target_sign_is_bit_identical(cid, dtype):
    """Negating every target quaternion gives the same bits of e and J."""
    c = _case(cid)
    q, ft, pt = _inputs(cid)["in64"] if dtype == torch.float64 else _inputs(cid)["in32"]
    neg = ft.copy()
    neg[..., :4] *= -1
    prob = _problem(cid)
    a = prob.fk_jac(_t(q, dtype), _t(ft, dtype), _t(pt, dtype), None, dt=c["wl"]["dt"])
    b = prob.fk_jac(_t(q, dtype), _t(neg, dtype), _t(pt, dtype), None, dt=c["wl"]["dt"])
    assert torch.equal(a[0], b[0]) and torch.equal(a[1], b[1])


# ---- step: the packed K1 form -------------------------------------------------------------------------------------------
@pytest.mark.parametrize("cid", list(LIE_CASES))
def test_step_on_large_rotations_against_oracle(cid):
    """bik_step (fp32, packed rows) and bik_step64 on the grid's targets against Oracle.step on identical inputs, with the
    bars of tests/test_gpu_k2_sizes.py (1e-4 and 2e-7 of max(1, |dq|)).  fp32 leaves out the instances next to the identity
    switch: there the fp32 e decides the side (test_fk_jac_against_mpmath checks J on the kernel's side), and across the
    switch Mi jumps by ~|v| / 2, so dq moves by ~2e-3 on the 0.3 m offsets."""
    c = _case(cid)
    inp = _inputs(cid)
    kw = dict(dt=c["wl"]["dt"], damping=c["wl"]["damping"])
    prob = _problem(cid)
    for dtype, key, tol in ((torch.float32, "in32", 1e-4), (torch.float64, "in64", 2e-7)):
        ref = c["orc"].step(*inp[key], None, **kw)
        assert not ref[2].any()
        dq, st = prob.step(*(_t(a, dtype) for a in inp[key]), None, **kw)
        assert int(st.max()) == 0 and int(st.min()) == 0
        keep = ~_straddle() if dtype == torch.float32 else np.ones(B, bool)
        err = np.abs(_np(dq)[keep] - ref[0][keep]).max()
        print(f"{cid}/{dtype}: max|dq - dq_oracle| {err:.2e} (|dq| up to {np.abs(ref[0]).max():.2f})")
        assert err <= tol * max(1.0, np.abs(ref[0]).max())


# ---- converge from far-away targets -------------------------------------------------------------------------------------
FAR_ANGLES = (2.5, 3.0, np.pi - 1e-2)
CONV = dict(max_iters=12, pos_threshold=2e-3, ori_threshold=2e-3)


@pytest.mark.parametrize("name", ["n7", "ur5e"])
def test_converge_from_far_targets_against_oracle(name):
    """bik_converge64: the oracle's iteration counts and flags, q within 1e-5; bik_converge: the oracle's flags on the fp32
    rounding of the inputs, q within 1e-3.  12 passes of 0.1 - 0.3 rad steps carry the K2 and oracle QP solutions'
    differences further than the converge64 tests' 1e-6 bar: 4.8e-6 on ur5e, 1.6e-7 on n7 (an H100)."""
    from mink_b200.engine import DeviceModel, Problem
    from oracle.ikoracle import Oracle

    _need_gpu()
    if name == "ur5e":
        wl, fm, spec, _ = load_case("ur5e")
        orc = Oracle(fm.to_blob(), spec, fm.nq, fm.nv)
        frames = task_frames(wl, fm)
    else:
        c = chain_case(7, seed=7)
        wl, fm, spec, orc, frames = c["wl"], c["fm"], c["spec"], c["orc"], c["frames"]
    prob = Problem(DeviceModel(fm, device=0), spec)
    fk = lambda qq: orc.fk(qq, frames)
    inp = make_inputs(fm, wl, B, fk, seed=8, sigma=0.3)
    rng = np.random.default_rng(51)
    poses, _ = fk(inp["q"])
    ft = np.zeros((B, 1, 7))
    for k, th in enumerate(FAR_ANGLES):
        idx = np.arange(k, B, len(FAR_ANGLES))
        ft[idx, 0] = targets_at_angle(poses[idx, 0], th, 0.05, rng)
    kw = dict(dt=wl["dt"], damping=wl["damping"])
    for dtype in (torch.float64, torch.float32):
        ins = (inp["q"], ft, inp["posture_target"]) if dtype == torch.float64 else tuple(_r32(a) for a in (inp["q"], ft, inp["posture_target"]))
        q_ref, it_ref, ok_ref, _ = orc.converge(*ins, None, **kw, **CONV)
        q = _t(ins[0], dtype)
        it, st = prob.converge(q, _t(ins[1], dtype), _t(ins[2], dtype), None, **kw, **CONV)
        it, st = it.cpu().numpy(), st.cpu().numpy()
        assert int((st & 15).max()) == 0
        np.testing.assert_array_equal((st & 16) == 0, ok_ref.astype(bool))
        err = np.abs(_np(q) - q_ref).max()
        print(f"{name}/{dtype}: converged {int(ok_ref.sum())}/{B}, {int((it != it_ref).sum())} iteration counts differ, "
              f"max|q - q_oracle| {err:.1e}")
        if dtype == torch.float64:
            np.testing.assert_array_equal(it, it_ref)
            assert err <= 1e-5
        else:
            assert err <= 1e-3


# ---- integrate ----------------------------------------------------------------------------------------------------------
INTEGRATE_NORMS = (0.0, 1e-16, 1e-8, 1.0, np.pi, 2 * np.pi - 1e-3, 5.0)


@pytest.mark.parametrize("dtype", [torch.float64, torch.float32], ids=["f64", "f32"])
@pytest.mark.parametrize("cid", ["free32", "ball64"])
def test_integrate_free_and_ball_joints(cid, dtype):
    """bik_integrate[64] with rotation steps |w| in INTEGRATE_NORMS (instance b takes norm b mod 7) on the free / ball joint:
    its quaternion against quat_integrate in extended precision, every other coordinate against q + dq."""
    c = _case(cid)
    fm = c["fm"]
    f64 = dtype == torch.float64
    kind = 0 if cid == "free32" else 1
    n = [i for i in range(fm.nnode) if int(fm.node_type[i]) == kind][0]
    qa, da = int(fm.node_qadr[n]) + 3 * (kind == 0), int(fm.node_dadr[n]) + 3 * (kind == 0)
    rng = np.random.default_rng(31)
    dq = rng.normal(0, 0.05, size=(B, fm.nv))
    ax = rng.normal(size=(B, 3))
    norms = np.array([INTEGRATE_NORMS[b % len(INTEGRATE_NORMS)] for b in range(B)])
    dq[:, da:da + 3] = norms[:, None] * ax / np.linalg.norm(ax, axis=1, keepdims=True)
    q = c["q"] if f64 else _r32(c["q"])
    dq = dq if f64 else _r32(dq)
    qt = _t(q, dtype)
    c["model"].integrate(qt, _t(dq, dtype))
    got = _np(qt)
    ref_q = lie_ref.quat_integrate(q[:, qa:qa + 4], dq[:, da:da + 3])
    lin = q.copy()
    for d in range(fm.nv):
        if int(fm.dof_qadr[d]) >= 0:
            lin[:, int(fm.dof_qadr[d])] += dq[:, d]
    if kind == 0:
        lin[:, qa - 3:qa] = q[:, qa - 3:qa] + dq[:, da - 3:da]
    rest = np.ones(fm.nq, bool)
    rest[qa:qa + 4] = False
    tol = 1e-15 if f64 else 4e-7
    dqn = np.abs(got[:, qa:qa + 4] - ref_q).max(1)
    print(f"{cid}/{'f64' if f64 else 'f32'}: max|quat - quat_ref| {dqn.max():.1e} at |w| = {norms[int(dqn.argmax())]:g}")
    assert dqn.max() <= tol
    assert np.abs(got[:, rest] - lin[:, rest]).max() <= 4 * tol
