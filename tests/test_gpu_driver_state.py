"""The device buffers a problem handle owns, across calls of different sizes and precisions.

bik_converge / bik_track keep a CUDA graph per problem and replay it while the call's arguments repeat.  The graph holds the
addresses of the K1 -> K2 hand-off and of the loop state; a bik_step on a larger batch, or an fp64 bik_step64 on the same
one, moves the hand-off.  The next bik_converge with the first call's arguments must run on the buffers the problem owns
now: same results as the first call, as a fresh handle and as the host-polled loop.
"""

import ctypes as C

import pytest

torch = pytest.importorskip("torch")
pytestmark = pytest.mark.gpu

from mink_b200 import _lib  # noqa: E402
from tests.test_gpu_track import CONV, _case, _equal, _graph_mode  # noqa: E402


@pytest.mark.parametrize("track", [False, True], ids=["converge", "track"])
@pytest.mark.parametrize("between", ["larger_step", "step64"])
def test_cached_converge_graph_follows_the_hand_off_buffers(between, track):
    from mink_b200.engine import Problem, _stream

    B, T = 100, 4
    c = _case("ur5e", B=B, T=T, seed=33)
    prob, kw = c["prob"], c["kw"]
    # the fp32 calls below size the hand-off for 4-byte elements, so that bik_step64 on the same batch has to move it
    assert "f32 for fp32 callers" in prob.describe(kw["damping"])
    q0 = torch.tensor(c["q0"], dtype=torch.float32, device="cuda:0")
    ft = c["ft"] if track else c["ft"][:, T - 1].contiguous()
    # Tensors allocated once and refilled in place: every call presents the same pointers, as a control loop does (the
    # Problem.converge / Problem.track wrappers allocate their outputs per call and would not reliably repeat them).
    q = torch.empty_like(q0)
    shape = (B, T) if track else (B,)
    iters = torch.empty(shape, dtype=torch.int32, device="cuda:0")
    status = torch.empty(shape, dtype=torch.int32, device="cuda:0")
    q_traj = torch.empty((B, T, c["fm"].nq), dtype=torch.float32, device="cuda:0")
    passes = torch.zeros(1, dtype=torch.int32, device="cuda:0")

    def run(p):
        q.copy_(q0); iters.fill_(-1); status.fill_(-1 if track else 0); q_traj.fill_(float("nan")); passes.zero_()
        inp, keep, _, _ = p._inputs(None, ft, c["pt"], None, dtype=torch.float32)
        loop = (float(kw["dt"]), float(kw["damping"]), CONV["max_iters"], CONV["pos_threshold"], CONV["ori_threshold"], 2)
        if track:
            _lib.check(p.lib.bik_track(p.handle, B, T, q.data_ptr(), C.byref(inp), None, *loop, q_traj.data_ptr(), iters.data_ptr(),
                                       status.data_ptr(), passes.data_ptr(), _stream()))
        else:
            _lib.check(p.lib.bik_converge(p.handle, B, q.data_ptr(), C.byref(inp), *loop, iters.data_ptr(), status.data_ptr(), _stream()))
        torch.cuda.synchronize()
        return [t.clone() for t in ((q, iters, status, q_traj, passes) if track else (q, iters, status))]

    first = run(prob)                                   # 1. hand-off and loop state sized for B, graph built and kept
    assert int(first[1].max()) > 0                      # (the loop did take steps)
    if between == "larger_step":                        # 2. the hand-off moves
        n = 10
        prob.step(q0.repeat(n, 1), c["ft"][:, 0].repeat(n, 1, 1), c["pt"].repeat(n, 1, 1), None, nsteps=2, integrate=True, **kw)
    else:
        prob.step(q0.double(), c["ft"][:, 0].double(), c["pt"].double(), None, nsteps=2, integrate=True, **kw)
    again = run(prob)                                   # 3. the arguments of 1.
    fresh = run(Problem(prob.model, c["spec"]))
    with _graph_mode("0"):
        polled = run(Problem(prob.model, c["spec"]))
    for other in (again, fresh, polled):
        for a, b in zip(first, other):
            _equal(a, b)
