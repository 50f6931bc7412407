"""K2 at the edges of its coupled-dof range, on the host emulation (one lane per instance), against the fp64 oracle.

The golden robots couple 6, 7, 18, 20-25, 31 and 43 dofs.  K2 switches instantiation at other sizes: 8 / 9 (G = 4 -> 8 lanes
per problem), 32 / 33 (32-bit -> 64-bit active-set masks), 64 (the widest block), and on the general path at nu + 1 = 8, 16,
32, 64, 65 (lanes per problem, then slots per lane).  Synthetic hinge chains (tests/helpers.chain_case) put a problem on
each side of every switch; each case first checks that it really sits where it claims, and that the oracle's optimum has
the last coupled dof at a bound in some instances and free in others, so the top mask bit and the top slot matter.
tests/test_gpu_k2_sizes.py runs the same cases through the CUDA kernels.
"""

import functools

import numpy as np
import pytest
from scipy.optimize import nnls

from mink_b200.workloads import make_inputs
from tests.emu_lib import Emu
from tests.helpers import CHAIN_CASES as ALL_CASES, assert_chain_uses_top_of_block, chain_case_by_id

B = 48


def paths_for(nu, collision):
    """The K2 paths the emulation runs at this size: 1 general, 3 small-group (32-bit masks), 8 small-group (64-bit masks)."""
    if collision:
        return [1]
    return [1] + ([3] if nu <= 32 else []) + [8]


@functools.lru_cache(maxsize=None)
def case(cid):
    c = chain_case_by_id(cid)
    fm, wl = c["fm"], c["wl"]
    inp = make_inputs(fm, wl, B, c["fk"], seed=5, sigma=0.3)
    r32 = lambda a: np.asarray(a, np.float32).astype(np.float64)
    c["in64"] = (inp["q"], inp["frame_targets"], inp["posture_target"])
    c["in32"] = tuple(r32(a) for a in c["in64"])
    c["emu"] = Emu(fm.to_blob(), c["spec"], fm.nq, fm.nv)
    c["ref64"] = c["orc"].step(*c["in64"], None, dt=wl["dt"], damping=wl["damping"])
    c["ref32"] = c["orc"].step(*c["in32"], None, dt=wl["dt"], damping=wl["damping"])
    return c


@pytest.mark.parametrize("cid", list(ALL_CASES))
def test_case_sits_on_its_boundary(cid):
    """The case couples the dofs it claims (nu, and nfree unbounded leading ones), and the oracle's optimum uses the top of
    the coupled block."""
    kw, nu, nfree = ALL_CASES[cid]
    c = case(cid)
    h = c["emu"].header()
    assert (h["nu"], h["nfree"]) == (nu, nfree), h
    assert_chain_uses_top_of_block(c, nu, c["in64"][0], c["ref64"])
    nact = c["ref64"][3]
    print(f"{cid}: nq={c['fm'].nq} nv={c['fm'].nv} nu={h['nu']} nfree={h['nfree']} active mean {nact.mean():.1f} max {nact.max()}")


@pytest.mark.parametrize("cid,path", [(cid, p) for cid, (kw, nu, _) in ALL_CASES.items() for p in paths_for(nu, kw.get("collision", False))])
def test_k2_paths_match_oracle(cid, path):
    """The step forms the driver launches, on identical inputs: packed fp32 rows with fp32 I/O (bik_step's form), and packed
    fp64 rows with fp64 I/O (bik_step64's)."""
    c = case(cid)
    emu, wl, h = c["emu"], c["wl"], c["emu"].header()
    dt, damping = wl["dt"], wl["damping"]
    nact = c["ref64"][3]
    errs = []
    for prec, ref, inp, tol in (("f32", c["ref32"], c["in32"], 1e-4), ("f64", c["ref64"], c["in64"], 2e-7)):
        q, ft, pt = inp
        dq_ref = ref[0]
        pk, Gc, hc = emu.fk_jac(q, ft, pt, None, dt=dt, prec=prec, packed=True)
        dq, st, it, *_ = emu.solve(q, None, None, None, Gc, hc, dt, damping, use_double=path, io64=prec == "f64", pk=pk, ptgt=pt)
        assert not st.any(), (prec, np.unique(st))
        err = np.abs(dq - dq_ref).max()
        errs.append(err)
        assert err < tol * max(1.0, np.abs(dq_ref).max()), (prec, err)
    print(f"{cid} path {path}: nu={h['nu']} nfree={h['nfree']} active mean {nact.mean():.1f} max|dq - dq_oracle| fp32 {errs[0]:.2e} fp64 {errs[1]:.2e}")


def check_kkt(x, H, c, lo, hi, G=None, h=None, tol_rel=1e-6):
    """Optimality of x for min 1/2 x'Hx + c'x, lo <= x <= hi (, G x <= h) without a QP solver: x feasible; non-negative
    multipliers of the active general rows, recovered by least squares on the dofs away from their bounds, cancel the gradient
    there; at the bounds what remains of it points outwards.  Returns the largest multiplier."""
    B, n = x.shape
    worst = 0.0
    for b in range(B):
        tol = tol_rel * max(1.0, np.abs(H[b]).max()) * max(1.0, np.abs(x[b]).max())
        assert np.all(x[b] >= lo[b] - 1e-9) and np.all(x[b] <= hi[b] + 1e-9), b
        g = H[b] @ x[b] + c[b]
        at_lo, at_hi = x[b] <= lo[b] + 1e-9, x[b] >= hi[b] - 1e-9
        free = ~(at_lo | at_hi)
        if G is not None and G.shape[1]:
            fin = np.isfinite(h[b])
            Gb, hb = G[b][fin], h[b][fin]
            r = Gb @ x[b] - hb
            assert np.all(r <= 1e-9 * max(1.0, np.abs(hb).max(initial=0.0))), (b, r.max())
            act = np.abs(r) <= 1e-8 * max(1.0, np.abs(hb).max(initial=0.0))
            if act.any():
                A = Gb[act]   # active rows may be dependent on the free dofs: non-negative least squares picks a valid set
                mu = nnls(A[:, free].T, -g[free])[0]
                g = g + A.T @ mu
                worst = max(worst, float(mu.max()))
        assert np.all(np.abs(g[free]) <= tol), (b, np.abs(g[free]).max(), tol)
        assert np.all(g[at_lo & ~at_hi] >= -tol) and np.all(g[at_hi & ~at_lo] <= tol), b
    return worst


@pytest.mark.parametrize("cid", list(ALL_CASES))
def test_objective_box_and_optimality(cid):
    """The emulation's own H, c, lo, hi (general path, fp64 rows) against the oracle's, then the fp64 dq checked against
    those: feasible, and optimal by the KKT conditions -- a check that does not rest on the oracle's QP solver."""
    c = case(cid)
    emu, orc, wl, fm = c["emu"], c["orc"], c["wl"], c["fm"]
    dt, damping = wl["dt"], wl["damping"]
    q, ft, pt = c["in64"]
    J, e, ep, Gc, hc = emu.fk_jac(q, ft, pt, None, dt=dt, prec="f64")
    Jr, er, epr = orc.fk_jac(q, ft, pt, None)
    np.testing.assert_allclose(J, Jr, atol=1e-9)
    np.testing.assert_allclose(e, er, atol=1e-10)
    np.testing.assert_allclose(ep, epr, atol=1e-12)
    if c["spec"].npairs:
        Gr, hr = orc.collision(q, dt)
        fin = np.isfinite(hr)
        assert np.array_equal(np.isfinite(hc), fin) and 0.3 < fin.any(axis=1).mean() < 1.0
        np.testing.assert_allclose(hc[fin], hr[fin], rtol=1e-9, atol=1e-9)
        np.testing.assert_allclose(Gc, Gr, atol=1e-9)
    pk, Gc, hc = emu.fk_jac(q, ft, pt, None, dt=dt, prec="f64", packed=True)
    dq, st, it, H, cv, lo, hi = emu.solve(q, None, None, None, Gc, hc, dt, damping, use_double=1, io64=True, want_objective=True, pk=pk, ptgt=pt)
    assert not st.any()
    Hr, cr = orc.objective(Jr, er, epr, damping)
    np.testing.assert_allclose(H, Hr, atol=1e-8 * np.abs(Hr).max())   # costs and gains are kept in fp32
    np.testing.assert_allclose(cv, cr, atol=1e-8 * max(1.0, np.abs(cr).max()))
    lor, hir = orc.box(q, dt)
    for a, r in ((lo, lor), (hi, hir)):
        fin = np.isfinite(r)
        assert np.array_equal(np.isfinite(a), fin)
        np.testing.assert_allclose(a[fin], r[fin], atol=1e-6)
    mu = check_kkt(dq, H, cv, lo, hi, Gc if c["spec"].npairs else None, hc if c["spec"].npairs else None)
    print(f"{cid}: nu={emu.header()['nu']} KKT holds on {len(dq)} instances, largest collision multiplier {mu:.3g}")
