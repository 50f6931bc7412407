"""Every K2 instantiation at the edges of its coupled-dof range, through the CUDA kernels, against the fp64 oracle.

The synthetic chains of tests/helpers.CHAIN_CASES sit on both sides of every switch of K2's dispatch (tests/test_k2_sizes_cpu.py
checks the same cases on the host emulation, where every kernel runs with one lane).  Here the lane distribution, the
shuffles, the slots per lane and the problems per warp are the device's:
  * small-group path (box limits only): G = 4 up to nu = 8, G = 8 from nu = 9, 64-bit active-set masks from nu = 33, each in
    its three I/O forms -- bik_step (packed fp32 rows), bik_solve (dense fp32 rows), bik_solve64 / bik_step64 (fp64);
  * general path (collision rows, BIK_K2_PATH=dense, bik_qp_objective, bik_limits_box): W = 8, 16, 32 lanes per problem for
    nu + 1 <= 8, 16, 32, then 2 slots per lane up to nu + 1 = 64 and 3 at nu = 64;
each case first checks, through bik_problem_describe, that its solving launch takes the instantiation it is there for; then
it runs on batches of one problem, one less and one more than a CTA's problems, and more than two resident waves of the persistent
grid (the tile loops and the dynamic tile counter wrap).  K1 runs on the same chains: nq = 1 ... 65, ragged batches, inputs
that start one row into their buffer (the bulk-copy alignment check takes its plain-load fallback).
"""

import contextlib
import functools
import os

import numpy as np
import pytest

torch = pytest.importorskip("torch")
pytestmark = pytest.mark.gpu

from mink_b200.workloads import make_inputs  # noqa: E402
from tests.helpers import CHAIN_CASES, assert_chain_uses_top_of_block, chain_case_by_id  # noqa: E402

SIGMA = 0.3


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


def _collision(cid):
    return CHAIN_CASES[cid][0].get("collision", False)


# ---- cases, problems, inputs --------------------------------------------------------------------------------------------
@functools.lru_cache(maxsize=None)
def _case(cid):
    from mink_b200.engine import DeviceModel

    _need_gpu()
    c = chain_case_by_id(cid)
    c["model"] = DeviceModel(c["fm"], device=0)   # one model per case; K2 knobs are read per problem
    return c


def _problem(cid, env=None, model=None):
    from mink_b200.engine import Problem

    c = _case(cid)
    with _env(env or {}):
        return Problem(model or c["model"], c["spec"])


@functools.lru_cache(maxsize=None)
def _inputs(cid, B):
    """Inputs in fp64 and their fp32 rounding, with the oracle's step on each (identical inputs)."""
    c = _case(cid)
    wl = c["wl"]
    inp = make_inputs(c["fm"], wl, B, c["fk"], seed=1000 + B, sigma=SIGMA)
    in64 = (inp["q"], inp["frame_targets"], inp["posture_target"])
    in32 = tuple(np.asarray(a, np.float32).astype(np.float64) for a in in64)
    kw = dict(dt=wl["dt"], damping=wl["damping"])
    ref64 = c["orc"].step(*in64, None, **kw)
    ref32 = c["orc"].step(*in32, None, **kw)
    assert not ref64[2].any() and not ref32[2].any()
    return dict(in64=in64, in32=in32, ref64=ref64, ref32=ref32)


# ---- where each launch lands --------------------------------------------------------------------------------------------
def _k2_name(cid, env):
    """What bik_problem_describe must call K2's solving path for this case under `env`."""
    kw, nu, nfree = CHAIN_CASES[cid]
    if _collision(cid) or env.get("BIK_K2_PATH") == "dense":
        rows = nu + 1   # k2_kernel<W, SLOTS>: W x SLOTS covers the coupled dofs and the right-hand side
        if rows <= 16:
            return f"general {8 if rows <= 8 else 16}-lanes-per-problem"
        return "general warp-per-problem" + ("" if rows <= 32 else f", {(rows + 31) // 32} slots per lane")
    if nu > 32:
        return "small-group G=8 (64-bit masks)"
    return f"small-group G={int(env.get('BIK_K2_GROUP', 8 if nu > 8 else 4))}"


def _device_limits():
    p = torch.cuda.get_device_properties(0)
    per_sm = getattr(p, "shared_memory_per_multiprocessor", 228 * 1024)
    per_cta = getattr(p, "shared_memory_per_block_optin", 227 * 1024)
    return p.multi_processor_count, per_sm, per_cta


def _tiles(cid, env):
    """(problems per CTA, an upper bound on the problems one resident wave of the persistent grid holds) of K2's solving launch.
    Small-group: 32 / G problems per warp, warps per CTA as the launcher picks them from the per-problem slot (bik_k2t.h
    k2t_slot_bytes; the frame task's columns are the nu coupled dofs here).  General: 32 / W problems per warp, 8 warps per CTA
    at most.  The wave is bounded by 64 resident warps and by the shared memory of an SM."""
    kw, nu, nfree = CHAIN_CASES[cid]
    fm = _case(cid)["fm"]
    nsm, smem_sm, smem_cta = _device_limits()
    name = _k2_name(cid, env)
    if name.startswith("small-group"):
        G = 4 if "G=4" in name else 8
        tri = lambda n: n * (n + 1) // 2
        union = max(tri(nu + 1), (6 * nu + 6) | 1, (fm.nq + fm.nv) | 1)
        slot = 8 * (tri(nu) + union + 3 * nu) + 8 * nu
        wb = (32 // G * slot + 15) & ~15
        nw = max(1, min(8, smem_cta // wb))
        ctas = max(1, min(64 // nw, smem_sm // (nw * wb + 1024)))
        return nw * 32 // G, nsm * ctas * nw * 32 // G
    lanes = 8 if "8-lanes" in name else (16 if "16-lanes" in name else 32)
    return 8 * 32 // lanes, nsm * 64 * 32 // lanes


def _envs(cid):
    """Default dispatch, the general kernel on every size, and the other small-group width where both apply."""
    nu = CHAIN_CASES[cid][1]
    if _collision(cid):
        return {"default": {}}
    envs = {"default": {}, "dense": {"BIK_K2_PATH": "dense"}}
    if nu <= 32:
        envs["group"] = {"BIK_K2_GROUP": 8 if nu <= 8 else 4}
    return envs


def _batches(cid):
    """B = 1, one less and one more than a CTA's problems under every env, and one ragged batch above two waves of them all."""
    small, wave = {1}, 0
    for env in _envs(cid).values():
        ppc, w = _tiles(cid, env)
        small |= {max(1, ppc - 1), ppc + 1}
        wave = max(wave, w)
    return sorted(small), 2 * wave + 5


ENTRY_PARAMS = [(cid, e) for cid in CHAIN_CASES for e in _envs(cid)]


def _check_dq(dq, st, ref, tol, what):
    assert int(st.max()) == 0 and int(st.min()) == 0, (what, np.unique(_np(st)))
    dq_ref = ref[0]
    err = np.abs(_np(dq) - dq_ref).max()
    assert err < tol * max(1.0, np.abs(dq_ref).max()), (what, err)
    return err


# ---- K2 -----------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("cid,envname", ENTRY_PARAMS)
def test_k2_entry_points_against_oracle(cid, envname):
    """bik_step (fp32: packed rows), bik_solve on the oracle's J, e cast to fp32 (dense fp32 rows), bik_solve64 and bik_step64
    (fp64) against the oracle on identical inputs, at every batch of _batches; repeated calls are bit-identical."""
    env = _envs(cid)[envname]
    kw, nu, nfree = CHAIN_CASES[cid]
    c = _case(cid)
    prob = _problem(cid, env)
    d = prob.describe(c["wl"]["damping"])
    assert f"k2: {_k2_name(cid, env)} f64" in d and f"coupled={nu} " in d, d
    if "small-group" in d:
        assert f"eliminated once: {nfree})" in d, d
    wl, orc = c["wl"], c["orc"]
    dt, damping = wl["dt"], wl["damping"]
    small, big = _batches(cid)
    assert_chain_uses_top_of_block(c, nu, _inputs(cid, big)["in64"][0], _inputs(cid, big)["ref64"])
    f32 = lambda a: torch.tensor(np.ascontiguousarray(a), dtype=torch.float32, device="cuda:0")
    f64 = lambda a: torch.tensor(np.ascontiguousarray(a), dtype=torch.float64, device="cuda:0")
    worst = np.zeros(4)
    for B in small + [big]:
        inp = _inputs(cid, B)
        q, ft, pt = map(f32, inp["in32"])
        dq, st = prob.step(q, ft, pt, None, dt=dt, damping=damping)
        worst[0] = max(worst[0], _check_dq(dq, st, inp["ref32"], 1e-4, ("step", B)))
        q8, ft8, pt8 = map(f64, inp["in64"])
        dq8, st8 = prob.step(q8, ft8, pt8, None, dt=dt, damping=damping)
        worst[1] = max(worst[1], _check_dq(dq8, st8, inp["ref64"], 2e-7, ("step64", B)))
        if B == big:
            for rep in range(2):   # the tile counter rewinds: the same call again gives the same bits
                dq2, _ = prob.step(q, ft, pt, None, dt=dt, damping=damping)
                assert torch.equal(dq, dq2), rep
            continue
        J, e, ep = orc.fk_jac(*inp["in64"], None)
        if c["spec"].npairs:
            Gc, hc = orc.collision(inp["in64"][0], dt)
        else:
            Gc, hc = np.zeros((B, 0, c["fm"].nv)), np.zeros((B, 0))
        dq, st = prob.solve(f32(inp["in64"][0]), f32(J), f32(e), f32(ep), f32(Gc), f32(hc), dt, damping)
        worst[2] = max(worst[2], _check_dq(dq, st, inp["ref64"], 1e-4, ("solve", B)))
        dq, st = prob.solve(q8, f64(J), f64(e), f64(ep), f64(Gc), f64(hc), dt, damping)
        worst[3] = max(worst[3], _check_dq(dq, st, inp["ref64"], 2e-7, ("solve64", B)))
    print(f"{cid}/{envname}: {d.split('; k2: ')[1]} nu={nu} nfree={nfree} B={small + [big]} max|dq - dq_oracle| "
          f"step {worst[0]:.2e} step64 {worst[1]:.2e} solve {worst[2]:.2e} solve64 {worst[3]:.2e}")


@pytest.mark.parametrize("cid", [cid for cid in CHAIN_CASES if not CHAIN_CASES[cid][0].get("collision")])
def test_static_tile_assignment_gives_the_same_bits(cid):
    """BIK_K2_DYNAMIC=0 (round-robin tiles) and the default atomic tile counter solve every instance the same way."""
    c = _case(cid)
    small, big = _batches(cid)
    inp = _inputs(cid, big)
    q, ft, pt = (torch.tensor(a, dtype=torch.float32, device="cuda:0") for a in inp["in32"])
    kw = dict(dt=c["wl"]["dt"], damping=c["wl"]["damping"])
    dq, st = _problem(cid).step(q, ft, pt, None, **kw)
    dq_s, st_s = _problem(cid, {"BIK_K2_DYNAMIC": 0}).step(q, ft, pt, None, **kw)
    assert int(st.max()) == 0 and torch.equal(st, st_s)
    assert torch.equal(dq, dq_s)


@pytest.mark.parametrize("cid", list(CHAIN_CASES))
def test_objective_and_box_against_oracle(cid):
    """bik_qp_objective[64] and bik_limits_box[64] always run on the general kernel, so at these sizes on every (W, SLOTS) of
    it, <32, 2> and <32, 3> included."""
    c = _case(cid)
    prob = _problem(cid)
    wl, orc = c["wl"], c["orc"]
    small, big = _batches(cid)
    B = small[-1]
    inp = _inputs(cid, B)
    J, e, ep = orc.fk_jac(*inp["in64"], None)
    Hr, cr = orc.objective(J, e, ep, wl["damping"])
    scale = np.abs(Hr).max()
    # fp32: the rows' rounding (tolerances of the golden K2 tests); fp64: costs and gains are kept in fp32
    for dtype, tol_H, tol_c in ((torch.float32, 1e-6, 1e-5), (torch.float64, 1e-8, 1e-8)):
        t = lambda a: torch.tensor(np.ascontiguousarray(a), dtype=dtype, device="cuda:0")
        H, cv = prob.objective(t(J), t(e), t(ep), wl["damping"])
        np.testing.assert_allclose(_np(H), Hr, atol=tol_H * scale)
        np.testing.assert_allclose(_np(cv), cr, atol=tol_c * max(1.0, np.abs(cr).max()))
        q = inp["in32"][0] if dtype == torch.float32 else inp["in64"][0]
        lo, hi = prob.box(t(q), wl["dt"])
        lor, hir = orc.box(q, wl["dt"])
        for a, r in ((_np(lo), lor), (_np(hi), hir)):
            fin = np.isfinite(r)
            assert np.array_equal(np.isfinite(a), fin)
            np.testing.assert_allclose(a[fin], r[fin], atol=1e-6)


# ---- K1 at the same sizes -----------------------------------------------------------------------------------------------
K1_CASES = ["n1", "n7", "n8", "n9", "n33", "n64", "ball64", "coll64"]   # nq = 1, 7, 8, 9, 33, 64, 65, and collision rows


def _check_k1(cid, out, inp, f64):
    J, e, ep, Gc, hc = map(_np, out)
    c = _case(cid)
    q = inp["in64"][0] if f64 else inp["in32"][0]
    Jr, er, epr = c["orc"].fk_jac(*(inp["in64"] if f64 else inp["in32"]), None)
    tJ, te, tp = (1e-9, 1e-10, 1e-12) if f64 else (5e-5, 2e-5, 1e-6)
    np.testing.assert_allclose(J, Jr, atol=tJ)
    np.testing.assert_allclose(e, er, atol=te)
    np.testing.assert_allclose(ep, epr, atol=tp)
    if c["spec"].npairs:
        Gr, hr = c["orc"].collision(q, c["wl"]["dt"])
        fin = np.isfinite(hr)
        assert np.array_equal(np.isfinite(hc), fin) and fin.any()
        np.testing.assert_allclose(hc[fin], hr[fin], **(dict(rtol=1e-9, atol=1e-9) if f64 else dict(rtol=2e-4, atol=2e-3)))
        np.testing.assert_allclose(Gc, Gr, atol=1e-9 if f64 else 2e-5)


@pytest.mark.parametrize("cid", K1_CASES)
def test_k1_against_oracle_and_bulk_copy_fallback(cid):
    """fk_jac in fp32 and fp64 against the oracle; then fk_jac and step with the bulk-copy input pipeline on and off
    (BIK_USE_TMA), on buffers that start at row 0 and at row 1 (q and targets no longer 16-byte aligned for odd nq): all
    bit-identical."""
    from mink_b200.engine import DeviceModel

    c = _case(cid)
    B = 3 * 64 + 37   # ragged against every lanes-per-instance choice
    inp = _inputs(cid, B)
    dt, damping = c["wl"]["dt"], c["wl"]["damping"]
    prob = _problem(cid)
    for dtype, key in ((torch.float32, "in32"), (torch.float64, "in64")):
        t = [torch.tensor(a, dtype=dtype, device="cuda:0") for a in inp[key]]
        _check_k1(cid, prob.fk_jac(t[0], t[1], t[2], None, dt=dt), inp, dtype == torch.float64)
    with _env({"BIK_USE_TMA": 0}):
        model_plain = DeviceModel(c["fm"], device=0)
    prob_plain = _problem(cid, model=model_plain)
    for dtype, key in ((torch.float32, "in32"), (torch.float64, "in64")):
        outs = []
        for p in (prob, prob_plain):
            for off in (0, 1):
                bufs = []
                for a in inp[key]:
                    a = np.asarray(a)
                    if a.ndim >= 2 and a.shape[0] == B:   # per-instance rows: place them one row into a larger buffer
                        big = torch.full((B + off,) + a.shape[1:], float("nan"), dtype=dtype, device="cuda:0")
                        big[off:] = torch.tensor(a, dtype=dtype)
                        bufs.append(big[off:])
                    else:
                        bufs.append(torch.tensor(a, dtype=dtype, device="cuda:0"))
                q, ft, pt = bufs
                res = list(p.fk_jac(q, ft, pt, None, dt=dt))
                dq, st = p.step(q, ft, pt, None, dt=dt, damping=damping)
                assert int(st.max()) == 0
                outs.append([r.clone() for r in res] + [dq.clone()])
        for o in outs[1:]:
            for a, b in zip(outs[0], o):
                assert torch.equal(a, b) or (a.numel() == 0 and b.numel() == 0)


@pytest.mark.parametrize("group", [1, 4, 32])
def test_k1_lane_groups_on_the_64_hinge_chain(group):
    """K1's lanes-per-instance mapping (BIK_K1_GROUP) on a 64-node serial chain, the longest lane program: the oracle's J, e."""
    from mink_b200.engine import DeviceModel

    c = _case("n64")
    with _env({"BIK_K1_GROUP": group}):
        model = DeviceModel(c["fm"], device=0)
    prob = _problem("n64", model=model)
    assert f"k1: {group} lanes/instance" in prob.describe(c["wl"]["damping"])
    inp = _inputs("n64", 263)
    t = [torch.tensor(a, dtype=torch.float32, device="cuda:0") for a in inp["in32"]]
    _check_k1("n64", prob.fk_jac(t[0], t[1], t[2], None, dt=c["wl"]["dt"]), inp, False)
