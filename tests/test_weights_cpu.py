"""Per-instance task weights (bik_converge_weighted / bik_track_weighted) through the pass loop compiled for the host
(tests/host_emu), no GPU needed.

A weight w multiplies a row of the packed J and e that K1 hands to K2, so instance b solves with the costs cost * w[b]:
all-ones weights give the unweighted results bit for bit, random weights give what the fp64 oracle gives with those costs,
zero weights on a frame task give the problem without that task, and out-of-range weights are clamped and flagged.
"""

import copy

import numpy as np
import pytest

from tests.emu_weights_lib import WeightedEmu
from tests.helpers import load_case, track_case

CONV = dict(max_iters=10, pos_threshold=2e-3, ori_threshold=2e-3)
BAD_WEIGHT = 32


def _row_blocks(spec):
    """[(task index, first row, rows)] of the frame and CoM tasks, in the stacked row order of J."""
    out, row = [], 0
    for i, t in enumerate(spec.tasks):
        k = {0: 6, 3: 6, 2: 3}.get(int(t.kind), 0)
        if k:
            out.append((i, row, k))
            row += k
    assert row == spec.nrows
    return out


def _weighted_spec(spec, w):
    """The problem with every frame / CoM cost multiplied by the instance's weights w [K]."""
    s = copy.deepcopy(spec)
    for i, r0, k in _row_blocks(spec):
        s.tasks[i].cost = np.asarray(s.tasks[i].cost, np.float64).copy()
        s.tasks[i].cost[:k] = s.tasks[i].cost[:k] * w[r0:r0 + k]
    return s


def _wemu(name, spec=None):
    """The weighted pass loops on the workload's problem (or on `spec`)."""
    wl, fm, spec0, g = load_case(name)
    return WeightedEmu(fm.to_blob(), spec0 if spec is None else spec, fm.nq, fm.nv)


def _eq(a, b):
    np.testing.assert_array_equal(a, b)


@pytest.mark.parametrize("dtype", [np.float32, np.float64])
@pytest.mark.parametrize("name", ["ur5e", "g1", "spot"])
def test_ones_are_the_identity(name, dtype):
    """ur5e: small-group K2; g1: three frame tasks; spot: CoM + collision rows, the general K2 path."""
    c = track_case(name, B=40 + 3, T=4, seed=3, dtype=dtype)
    emu, B, T, K = c["emu"], c["B"], c["T"], c["emu"].spec.nrows
    ct0 = None if c["ct"] is None else c["ct"][:, 0]
    ref = emu.converge(c["q0"], c["ft"][:, 0], c["pt"], ct0, **c["kw"], **CONV)
    wemu = _wemu(name)
    got = wemu.converge(c["q0"], c["ft"][:, 0], c["pt"], ct0, np.ones((B, K), dtype), **c["kw"], **CONV)
    for x, y in zip(got, ref):
        _eq(x, y)
    ln = np.random.default_rng(4).integers(0, T + 1, size=B).astype(np.int32)
    ref = emu.track(c["q0"], c["ft"], c["pt"], c["ct"], **c["kw"], **CONV, lengths=ln)
    got = wemu.track(c["q0"], c["ft"], c["pt"], c["ct"], np.ones((B, T, K), dtype), **c["kw"], **CONV, lengths=ln)
    for x, y in zip(got, ref):
        _eq(x, y)


@pytest.mark.parametrize("dtype", [np.float64, np.float32])
@pytest.mark.parametrize("name", ["ur5e", "g1", "spot"])
def test_weights_are_costs(name, dtype):
    """One step of instance b with weights w[b] is the fp64 oracle's step with the costs cost * w[b]: 1e-8 rad in fp64,
    1e-4 rad in fp32.  Then the whole loop: the same iteration counts as the oracle's loop with those costs."""
    from oracle.ikoracle import Oracle

    wl, fm, spec, g = load_case(name)
    c = track_case(name, B=6, T=1, seed=21, dtype=dtype)
    emu, B, K = _wemu(name), c["B"], spec.nrows
    w = np.random.default_rng(5).uniform(0.1, 1.0, size=(B, K))
    ft, ct = c["ft"][:, 0], None if c["ct"] is None else c["ct"][:, 0]
    q1, _, st = emu.converge(c["q0"], ft, c["pt"], ct, w.astype(dtype), **c["kw"], max_iters=1, pos_threshold=0.0, ori_threshold=0.0)
    assert not (st & ~16).any(), st
    qn, itn, _ = emu.converge(c["q0"], ft, c["pt"], ct, w.astype(dtype), **c["kw"], **CONV)
    f64 = lambda a: None if a is None else np.asarray(a, np.float64)
    tol = 1e-8 if dtype == np.float64 else 1e-4
    for b in range(B):
        orc = Oracle(fm.to_blob(), _weighted_spec(spec, w[b].astype(dtype).astype(np.float64)), fm.nq, fm.nv)
        args = (f64(c["q0"][b:b + 1]), f64(ft[b:b + 1]), f64(c["pt"][b:b + 1]), None if ct is None else f64(ct[b:b + 1]))
        _, q_ref, st_ref, _ = orc.step(*args, **c["kw"], nsteps=1, integrate=True)
        assert not st_ref.any()
        np.testing.assert_allclose(q1[b], q_ref[0], atol=tol, rtol=0)
        if dtype == np.float64:
            _, it_ref, _, _ = orc.converge(*args, **c["kw"], **CONV)
            assert itn[b] == it_ref[0], (b, itn[b], it_ref[0])


def _without_task(spec, drop):
    s = copy.deepcopy(spec)
    s.tasks = [t for i, t in enumerate(s.tasks) if i != drop]
    return s


@pytest.mark.parametrize("dtype", [np.float64, np.float32])
def test_zero_weights_remove_the_task(dtype):
    """G1's right foot weighted 0 in every instance: the problem without the right-foot task, to solver tolerance, with the
    same iteration counts (the task is out of the convergence test too); in track mode frame by frame as well."""
    from tests.emu_lib import Emu

    wl, fm, spec, g = load_case("g1")
    c = track_case("g1", B=24, T=3, seed=8, dtype=dtype, sigma=0.1)
    emu, B, T, K = _wemu("g1"), c["B"], c["T"], spec.nrows
    (i0, _, _), (i1, r1, _), _ = _row_blocks(spec)
    w = np.ones((B, T, K), dtype)
    w[:, :, r1:r1 + 6] = 0.0
    # the right foot's target is far away: with weight 1 the instance would chase it and fail the test
    ft = c["ft"].copy()
    ft[:, :, 1, 4:] += dtype(0.3)
    small = Emu(fm.to_blob(), _without_task(spec, i1), fm.nq, fm.nv)
    ft_small = np.delete(ft, 1, axis=2)
    conv = dict(max_iters=15, pos_threshold=1e-2, ori_threshold=1e-2)
    q, it, st = emu.converge(c["q0"], ft[:, 0], c["pt"], None, w[:, 0], **c["kw"], **conv)
    q_s, it_s, st_s = small.converge(c["q0"], ft_small[:, 0], c["pt"], None, **c["kw"], **conv)
    tol = 1e-9 if dtype == np.float64 else 1e-5
    np.testing.assert_allclose(q, q_s, atol=tol, rtol=0)
    _eq(it, it_s)
    _eq(st, st_s)
    assert (it < conv["max_iters"]).mean() >= 0.25, it
    _, q_traj, it, st, _ = emu.track(c["q0"], ft, c["pt"], None, w, **c["kw"], **conv)
    _, q_traj_s, it_s, st_s, _ = small.track(c["q0"], ft_small, c["pt"], None, **c["kw"], **conv)
    np.testing.assert_allclose(q_traj, q_traj_s, atol=10 * tol, rtol=0)
    _eq(it, it_s)
    _eq(st, st_s)


@pytest.mark.parametrize("dtype", [np.float32, np.float64])
def test_out_of_range_and_nan_weights_are_clamped_and_flagged(dtype):
    """Weights above 1, below 0 or NaN run as 1, 0 and 0, and only their instances get BIK_STATUS_BAD_WEIGHT."""
    c = track_case("spot", B=12, T=2, seed=9, dtype=dtype)
    emu, B, T, K = _wemu("spot"), c["B"], c["T"], c["emu"].spec.nrows
    rng = np.random.default_rng(10)
    w = rng.uniform(0.2, 1.0, size=(B, T, K)).astype(dtype)
    bad, clamped = w.copy(), w.copy()
    bad[1, :, 0], clamped[1, :, 0] = 1.5, 1.0
    bad[4, :, 7], clamped[4, :, 7] = -0.25, 0.0
    bad[7, :, K - 1], clamped[7, :, K - 1] = np.nan, 0.0
    bad[9, 1, 2], clamped[9, 1, 2] = np.inf, 1.0      # only frame 1 of instance 9
    flagged = np.zeros(B, bool)
    flagged[[1, 4, 7]] = True
    ct0 = c["ct"][:, 0]
    q, it, st = emu.converge(c["q0"], c["ft"][:, 0], c["pt"], ct0, bad[:, 0], **c["kw"], **CONV)
    q_c, it_c, st_c = emu.converge(c["q0"], c["ft"][:, 0], c["pt"], ct0, clamped[:, 0], **c["kw"], **CONV)
    _eq(q, q_c)
    _eq(it, it_c)
    assert not (st_c & BAD_WEIGHT).any()
    _eq(st, st_c | np.where(flagged, BAD_WEIGHT, 0))
    _, q_traj, it, st, _ = emu.track(c["q0"], c["ft"], c["pt"], c["ct"], bad, **c["kw"], **CONV)
    _, q_traj_c, it_c, st_c, _ = emu.track(c["q0"], c["ft"], c["pt"], c["ct"], clamped, **c["kw"], **CONV)
    _eq(q_traj, q_traj_c)
    _eq(it, it_c)
    flagged_t = np.repeat(flagged[:, None], T, axis=1)
    flagged_t[9, 1] = True
    _eq(st, st_c | np.where(flagged_t, BAD_WEIGHT, 0))
