"""Per-instance collision avoidance (bik_converge_coll / bik_track_coll) through the pass loops compiled for the host
(tests/host_emu/emu_collision.cpp), no GPU needed.

Instance b uses the CollisionAvoidanceLimit's pairs its mask enables, with its own minimum and detection distances: an
all-ones mask with the problem's distances gives the ..._bounded loops bit for bit, random masks and distances give what a
problem built with those pairs and distances gives bit for bit (and what the fp64 oracle gives), disabled pairs hand K2 a
zero row with h = +inf, an all-zero mask solves the QP without the limit, non-finite distances are flagged, and bik_track
with per-frame masks is one converge per frame.  Cases: ur5e_wall (floor and wall), Spot (feet against the floor and each
other), Go1 with its feet against the floor, and ALOHA with its 1 104 pairs.
"""

import copy

import numpy as np
import pytest

from mink_b200._abi import LIMIT_COLLISION
from mink_b200.workloads import WORKLOADS
from tests.emu_collision_lib import CollisionEmu
from tests.test_posture_weights_cpu import _at, _case, _eq, _lengths

CONV = dict(max_iters=10, pos_threshold=2e-3, ori_threshold=2e-3)
QP_MAXITER, NONFINITE = 2, 4
NAMES = ["ur5e_wall", "spot", "go1", "aloha_coll"]
GO1_FEET = dict(kind="collision", pairs=[(["FL", "FR", "RR", "RL"], ["floor"])], gain=0.85, minimum_distance=0.005,
                detection_distance=0.3, bound_relaxation=0.0)


def _workload(name):
    wl = WORKLOADS[name]
    if name == "go1":   # the workload has no collision limit: the feet against the floor
        return dict(wl, limits=list(wl["limits"]) + [GO1_FEET])
    return wl


def _ccase(name, dtype, B, T, seed):
    """tests.test_posture_weights_cpu._case on the plain workload (Go1 with its feet against the floor), with a CollisionEmu on
    its problem; lim: the spec's CollisionAvoidanceLimit."""
    c = _case(name, dtype, B, T, seed, wl=_workload(name))
    lim = next(l for l in c["spec"].limits if l.kind == LIMIT_COLLISION)
    fm = c["fm"]
    return dict(c, emu=CollisionEmu(fm.to_blob(), c["spec"], fm.nq, fm.nv), lim=lim, npairs=len(lim.pairs))


def _rebuilt(c, mask=None, dmin=None, ddet=None):
    """A CollisionEmu on the problem built with the pairs `mask` enables (in the same order) and the given distances."""
    s = copy.deepcopy(c["spec"])
    for l in s.limits:
        if l.kind == LIMIT_COLLISION:
            if mask is not None:
                l.pairs = l.pairs[np.asarray(mask, bool)]
            if dmin is not None:
                l.minimum_distance = float(dmin)
            if ddet is not None:
                l.detection_distance = float(ddet)
    fm = c["fm"]
    return CollisionEmu(fm.to_blob(), s, fm.nq, fm.nv), s


def _without_limit(spec):
    s = copy.deepcopy(spec)
    s.limits = [l for l in s.limits if l.kind != LIMIT_COLLISION]
    return s


def _random_masks(rng, B, npairs, density):
    m = rng.uniform(size=(B, npairs)) < density
    m[np.arange(B), rng.integers(0, npairs, size=B)] = True   # at least one pair per instance
    return m


def _random_distances(rng, lim, B, dtype):
    """fp32-representable distances around the problem's: dmin in [0, 2 dmin], ddet in [dmin + 0.01, 1.5 ddet]."""
    f32 = lambda a: a.astype(np.float32).astype(dtype)
    dmin = f32(rng.uniform(0.0, 2.0 * lim.minimum_distance + 1e-3, size=B))
    ddet = f32(dmin + rng.uniform(0.01, 1.5 * lim.detection_distance, size=B))
    return dmin, ddet


def _args(c, t=0):
    return c["q0"], c["ft"][:, t], c["pt"], _at(c["ct"], t)


@pytest.mark.parametrize("dtype", [np.float32, np.float64], ids=["f32", "f64"])
@pytest.mark.parametrize("name", NAMES)
def test_all_ones_mask_is_the_bounded_loop(name, dtype):
    """An all-ones mask with the problem's own distances gives the loops without collision arguments bit for bit, for converge
    and for track with ragged lengths; fp32 callers also with K1 forced to fp32 (BIK_K1_PRECISION=f32).  (The fp64 K1 of an
    fp32 caller uses the problem's distances in fp64, which fp32 inputs cannot restate: there the mask goes alone.)"""
    c = _ccase(name, dtype, B=12 + 3, T=3, seed=3)
    B, T, lim = c["B"], c["T"], c["lim"]
    ln = _lengths(B, T, 5)
    for f32k1 in ([False, True] if dtype == np.float32 else [False]):
        dist = dtype == np.float64 or f32k1
        co = (np.ones((B, c["npairs"]), bool), np.full(B, lim.minimum_distance, dtype) if dist else None,
              np.full(B, lim.detection_distance, dtype) if dist else None)
        cot = (np.ones((B, T, c["npairs"]), bool), np.full((B, T), lim.minimum_distance, dtype) if dist else None,
               np.full((B, T), lim.detection_distance, dtype) if dist else None)
        for x, y in zip(c["emu"].converge(*_args(c), co, **c["kw"], **CONV, f32k1=f32k1),
                        c["emu"].converge(*_args(c), None, **c["kw"], **CONV, f32k1=f32k1)):
            _eq(x, y)
        for x, y in zip(c["emu"].track(c["q0"], c["ft"], c["pt"], c["ct"], cot, **c["kw"], **CONV, lengths=ln, f32k1=f32k1),
                        c["emu"].track(c["q0"], c["ft"], c["pt"], c["ct"], None, **c["kw"], **CONV, lengths=ln, f32k1=f32k1)):
            _eq(x, y)


@pytest.mark.parametrize("dtype", [np.float32, np.float64], ids=["f32", "f64"])
@pytest.mark.parametrize("name", NAMES)
def test_random_masks_are_the_rebuilt_problem(name, dtype):
    """Each instance with a random mask (at least one pair) equals, bit for bit, the problem built with its enabled pairs: q,
    iterations, status, where neither run is flagged BIK_STATUS_QP_MAXITER (the one documented difference: the iteration cap
    counts the problem's pairs).  In fp64 one step also matches the fp64 oracle built with those pairs (1e-6 rad)."""
    from oracle.ikoracle import Oracle

    c = _ccase(name, dtype, B=8, T=1, seed=21)
    B, fm = c["B"], c["fm"]
    mask = _random_masks(np.random.default_rng(22), B, c["npairs"], 0.5)
    q, it, st = c["emu"].converge(*_args(c), (mask, None, None), **c["kw"], **CONV)
    q1, _, st1 = c["emu"].converge(*_args(c), (mask, None, None), **c["kw"], max_iters=1, pos_threshold=0.0, ori_threshold=0.0)
    compared = 0
    for b in range(B):
        emu_b, spec_b = _rebuilt(c, mask[b])
        sl = slice(b, b + 1)
        pt_b = None if c["pt"] is None else c["pt"][sl]
        ct = _at(c["ct"], 0)
        ct_b = None if ct is None else ct[sl]
        qr, itr, str_ = emu_b.converge(c["q0"][sl], c["ft"][sl, 0], pt_b, ct_b, None, **c["kw"], **CONV)
        if (st[b] | str_[0]) & QP_MAXITER:
            continue
        compared += 1
        _eq(q[b], qr[0]); _eq(it[b], itr[0]); _eq(st[b], str_[0])
        if dtype == np.float64 and not (st1[b] & ~16):
            orc = Oracle(fm.to_blob(), spec_b, fm.nq, fm.nv)
            f64 = lambda a: None if a is None else np.asarray(a, np.float64)
            _, q_ref, st_ref, _ = orc.step(f64(c["q0"][sl]), f64(c["ft"][sl, 0]), f64(pt_b), f64(ct_b), **c["kw"], nsteps=1, integrate=True)
            if not st_ref.any():
                np.testing.assert_allclose(q1[b], q_ref[0], atol=1e-6, rtol=0)
    assert compared >= B // 2


@pytest.mark.parametrize("dtype", [np.float32, np.float64], ids=["f32", "f64"])
@pytest.mark.parametrize("name", NAMES)
def test_random_distances_are_the_rebuilt_problem(name, dtype):
    """Random fp32-representable per-instance distances equal, bit for bit, problems built with those distances."""
    c = _ccase(name, dtype, B=6, T=1, seed=31)
    B = c["B"]
    dmin, ddet = _random_distances(np.random.default_rng(32), c["lim"], B, dtype)
    q, it, st = c["emu"].converge(*_args(c), (None, dmin, ddet), **c["kw"], **CONV)
    for b in range(B):
        emu_b, _ = _rebuilt(c, None, dmin[b], ddet[b])
        sl = slice(b, b + 1)
        ct = _at(c["ct"], 0)
        qr, itr, str_ = emu_b.converge(c["q0"][sl], c["ft"][sl, 0], None if c["pt"] is None else c["pt"][sl], None if ct is None else ct[sl],
                                       None, **c["kw"], **CONV)
        if (st[b] | str_[0]) & QP_MAXITER:
            continue
        _eq(q[b], qr[0]); _eq(it[b], itr[0]); _eq(st[b], str_[0])


@pytest.mark.parametrize("name", NAMES)
def test_disabled_pairs_hand_off_nothing(name):
    """K1's hand-off: a disabled pair is a zero G row with h = +inf, an enabled one is the row the full problem computes."""
    c = _ccase(name, np.float64, B=16, T=1, seed=41)
    B, npairs = c["B"], c["npairs"]
    mask = _random_masks(np.random.default_rng(42), B, npairs, 0.3)
    Gc, hc, st = c["emu"].k1(*_args(c), (mask, None, None), c["kw"]["dt"])
    G1, h1, st1 = c["emu"].k1(*_args(c), None, c["kw"]["dt"])
    assert np.isinf(hc[~mask]).all() and (hc[~mask] > 0).all()
    assert (Gc[~mask] == 0).all()
    _eq(hc[mask], h1[mask]); _eq(Gc[mask], G1[mask]); _eq(st, st1)
    assert np.isfinite(h1).any(), "no pair inside the detection distance: the case does not exercise the rows"


@pytest.mark.parametrize("name", NAMES)
def test_all_zero_mask_is_the_problem_without_the_limit(name):
    """No enabled pair: one fp64 step solves the QP without collision rows, as the oracle of the problem built without the
    limit does (to solver tolerance: the paths differ)."""
    from oracle.ikoracle import Oracle

    c = _ccase(name, np.float64, B=8, T=1, seed=51)
    B, fm = c["B"], c["fm"]
    q1, _, st = c["emu"].converge(*_args(c), (np.zeros((B, c["npairs"]), bool), None, None), **c["kw"], max_iters=1, pos_threshold=0.0,
                                  ori_threshold=0.0)
    orc = Oracle(fm.to_blob(), _without_limit(c["spec"]), fm.nq, fm.nv)
    ct = _at(c["ct"], 0)
    _, q_ref, st_ref, _ = orc.step(c["q0"], c["ft"][:, 0], c["pt"], ct, **c["kw"], nsteps=1, integrate=True)
    ok = (st_ref == 0) & ((st & ~16) == 0)
    assert ok.sum() >= B // 2
    np.testing.assert_allclose(q1[ok], q_ref[ok], atol=1e-6, rtol=0)


@pytest.mark.parametrize("dtype", [np.float32, np.float64], ids=["f32", "f64"])
@pytest.mark.parametrize("name", ["ur5e_wall", "spot"])
def test_nonfinite_distances_are_flagged(name, dtype):
    """A NaN or infinite distance falls back to the problem's value and sets BIK_STATUS_NONFINITE on that instance only."""
    c = _ccase(name, dtype, B=6, T=1, seed=61)
    B, lim = c["B"], c["lim"]
    dmin, ddet = np.full(B, lim.minimum_distance, dtype), np.full(B, lim.detection_distance, dtype)
    dmin[1] = np.nan
    ddet[2] = np.inf
    dmin[4] = -np.inf
    q, it, st = c["emu"].converge(*_args(c), (None, dmin, ddet), **c["kw"], **CONV)
    q_n, it_n, st_n = c["emu"].converge(*_args(c), None, **c["kw"], **CONV)
    _eq(q, q_n); _eq(it, it_n)
    assert not (st_n & NONFINITE).any()
    flagged = np.isin(np.arange(B), [1, 2, 4])
    _eq(st[~flagged], st_n[~flagged])
    _eq(st[flagged], st_n[flagged] | NONFINITE)


@pytest.mark.parametrize("dtype", [np.float32, np.float64], ids=["f32", "f64"])
@pytest.mark.parametrize("name", NAMES)
def test_track_equals_per_frame_converge(name, dtype):
    """bik_track_coll with a mask and distances per instance and frame equals one collision converge per frame, bit for bit,
    with ragged lengths; a NaN distance on one frame is flagged on that frame."""
    c = _ccase(name, dtype, B=12 + 5, T=3, seed=12)
    B, T, npairs = c["B"], c["T"], c["npairs"]
    rng = np.random.default_rng(13)
    mask = _random_masks(rng, B * T, npairs, 0.5).reshape(B, T, npairs)
    mask[::4, 1] = False   # no pair at all on some frames
    dmin, ddet = _random_distances(rng, c["lim"], B * T, dtype)
    dmin, ddet = dmin.reshape(B, T), ddet.reshape(B, T)
    dmin[5, 2] = np.nan
    ln = _lengths(B, T, 2)
    q = c["q0"]
    q_loop, it_loop, st_loop = np.zeros((B, T, c["fm"].nq), q.dtype), np.zeros((B, T), np.int32), np.zeros((B, T), np.int32)
    for t in range(T):
        q, it_loop[:, t], st_loop[:, t] = c["emu"].converge(q, c["ft"][:, t], c["pt"], _at(c["ct"], t), (mask[:, t], dmin[:, t], ddet[:, t]),
                                                            **c["kw"], **CONV)
        q_loop[:, t] = q
    q_end, q_traj, it, st, _ = c["emu"].track(c["q0"], c["ft"], c["pt"], c["ct"], (mask, dmin, ddet), **c["kw"], **CONV, lengths=ln)
    has = np.arange(T)[None, :] < ln[:, None]
    _eq(q_traj[has], q_loop[has])
    _eq(it[has], it_loop[has])
    _eq(st[has], st_loop[has])
    if ln[5] == T:
        assert st[5, 2] & NONFINITE and not (st[5, :2] & NONFINITE).any()
    q_ref = np.where(ln[:, None] > 0, q_loop[np.arange(B), np.maximum(ln - 1, 0)], c["q0"])
    _eq(q_end, q_ref)
