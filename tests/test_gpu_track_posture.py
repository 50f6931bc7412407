"""bik_track with a posture target sequence (bik_inputs.posture_batched = BIK_POSTURE_SEQ_SHARED / _BATCHED) and
track_ik with {posture_task: sequence}.

The definition: for every instance b, the results equal bik_converge called on frames 0..lengths[b]-1 in turn, each call
with frame t's posture target as an ordinary target -- bit for bit, through every track entry point and both loop modes.
Targets and sequences come from tests/test_track_posture_cpu.py's seeded cases.
"""

import ctypes as C
import os

import numpy as np
import pytest

torch = pytest.importorskip("torch")
pytestmark = pytest.mark.gpu

from mink_b200.workloads import WORKLOADS  # noqa: E402
from tests.test_track_posture_cpu import CONV, _case  # noqa: E402

DT = {np.float32: torch.float32, np.float64: torch.float64}


def _need_gpu():
    if not torch.cuda.is_available():
        pytest.skip("no CUDA device")


def _gpu_case(name, dtype, B, T, seed, wl=None):
    _need_gpu()
    from mink_b200._abi import spec_from_workload
    from mink_b200.engine import DeviceModel, Problem
    from mink_b200.workloads import load_flat

    c = _case(name, dtype, B=B, T=T, seed=seed, wl=wl)
    wl = wl or WORKLOADS[name]
    fm = load_flat(wl["robot"])
    c["fm"], c["spec"] = fm, spec_from_workload(fm, wl)
    c["model"] = DeviceModel(fm, device=0)
    c["prob"] = Problem(c["model"], c["spec"])
    dev = lambda a: None if a is None else torch.tensor(np.ascontiguousarray(a), dtype=DT[dtype], device="cuda:0")
    c["d"] = dict(ft=dev(c["ft"]), ct=dev(c["ct"]), pseq=dev(c["pseq"]))
    c["dev"] = dev
    return c


def _equal(a, b):
    torch.testing.assert_close(a, b, rtol=0, atol=0, equal_nan=True)


class _graph_mode:
    def __init__(self, mode):
        self.mode = mode

    def __enter__(self):
        os.environ["BIK_CONVERGE_GRAPH"] = self.mode

    def __exit__(self, *a):
        os.environ.pop("BIK_CONVERGE_GRAPH", None)


def _per_frame(c, prob, pts, w=None):
    """The definition's loop: one Problem.converge per frame on the same q; pts(t) is frame t's posture target."""
    d = c["d"]
    q = c["dev"](c["q0"])
    qs, its, sts = [], [], []
    for t in range(c["T"]):
        it, st = prob.converge(q, d["ft"][:, t], pts(t), None if d["ct"] is None else d["ct"][:, t], **c["kw"], **CONV,
                               weights=None if w is None else w[:, t])
        qs.append(q.clone()); its.append(it.clone()); sts.append(st.clone())
    return torch.stack(qs, 1), torch.stack(its, 1), torch.stack(sts, 1), q


def _track(c, prob, pt, posture_seq, lengths=None, w=None, **kw):
    d = c["d"]
    q = c["dev"](c["q0"])
    q_traj, it, st, passes = prob.track(q, d["ft"], pt, d["ct"], lengths=lengths, **c["kw"], **CONV, weights=w,
                                        posture_seq=posture_seq, **kw)
    return q_traj, it, st, q


def _check(loop, out, ln):
    q_loop, it_loop, st_loop, _ = loop
    q_traj, it, st, q = out
    has = torch.arange(q_traj.shape[1], device="cuda:0")[None, :] < ln[:, None]
    _equal(q_traj[has], q_loop[has])
    _equal(it[has], it_loop[has])
    _equal(st[has], st_loop[has])
    last = q_loop[torch.arange(q.shape[0], device="cuda:0"), (ln - 1).clamp(min=0).long()]
    _equal(q[ln > 0], last[ln > 0])


@pytest.mark.parametrize("dtype", [np.float32, np.float64], ids=["f32", "f64"])
@pytest.mark.parametrize("mode", ["1", "0"])
@pytest.mark.parametrize("name", ["ur5e", "g1", "h1", "tidybot", "ur5e_wall"])
def test_sequence_equals_per_frame_converge(name, mode, dtype):
    """bik_track / bik_track64 (form 3 against per-instance targets, form 2 against a shared one) and bik_track_weighted[64]
    (form 3 with random per-frame weights) against one bik_converge[_weighted][64] call per frame.  Graph mode ("1") and the
    host-polled loop ("0")."""
    c = _gpu_case(name, dtype, B=256 + 5, T=6, seed=12)
    B, T = c["B"], c["T"]
    ln = np.random.default_rng(2).integers(0, T + 1, size=B).astype(np.int32)
    ln[:3] = [0, T, 1]
    ln = torch.tensor(ln, device="cuda:0")
    seq, prob = c["d"]["pseq"], c["prob"]
    w = torch.tensor(np.random.default_rng(4).uniform(0.2, 1.0, size=(B, T, c["spec"].nrows)), dtype=DT[dtype], device="cuda:0")
    with _graph_mode(mode):
        _check(_per_frame(c, prob, lambda t: seq[:, t]), _track(c, prob, seq, True, ln, check_every=3), ln)
        shared = seq[7].contiguous()
        _check(_per_frame(c, prob, lambda t: shared[t]), _track(c, prob, shared, True, ln), ln)
        _check(_per_frame(c, prob, lambda t: seq[:, t], w=w), _track(c, prob, seq, True, ln, w=w), ln)


def test_track64_sequence_against_oracle():
    """bik_track64 with a per-instance sequence against the C oracle's converge loop run frame by frame with each frame's
    posture target: identical iteration counts, q within 1e-6."""
    c = _gpu_case("ur5e", np.float64, B=200 + 3, T=8, seed=44)
    q_traj, it, _, _ = _track(c, c["prob"], c["d"]["pseq"], True)
    q_traj, it = q_traj.cpu().numpy(), it.cpu().numpy()
    q = c["q0"].astype(np.float64)
    q_ref, it_ref = np.zeros_like(q_traj), np.zeros_like(it)
    for t in range(c["T"]):
        q, it_ref[:, t], _, _ = c["orc"].converge(q, c["ft"][:, t], c["pseq"][:, t], None, **c["kw"], **CONV)
        q_ref[:, t] = q
    print(f"track64 + posture sequence vs oracle: mismatching iters {int((it != it_ref).sum())}/{it.size}, "
          f"max|q - q_oracle| {np.abs(q_traj - q_ref).max():.2e}")
    np.testing.assert_array_equal(it, it_ref)
    np.testing.assert_allclose(q_traj, q_ref, atol=1e-6)


def test_graph_cache_follows_the_posture_form():
    """One problem handle, calls alternating between forms 0, 1, 2 and 3, two sequence buffers and two values of T, on fixed
    input and output buffers (so that a cached graph is replayed where the call is the same): each result equals the same call
    on a fresh problem, so no graph captured for another form, buffer or T is replayed."""
    from mink_b200 import _lib
    from mink_b200._abi import POSTURE_SEQ_BATCHED, POSTURE_SEQ_SHARED
    from mink_b200.engine import Problem, _stream

    c = _gpu_case("ur5e", np.float32, B=300 + 5, T=6, seed=55)
    B, nq, seq = c["B"], c["fm"].nq, c["d"]["pseq"]
    seq_b = (seq + 0.05).contiguous()
    fts = {6: c["d"]["ft"], 4: c["d"]["ft"][:, :4].contiguous()}
    q0 = c["dev"](c["q0"])
    calls = {
        "form0": (6, seq[0, 0].contiguous(), None),
        "form1": (6, seq[:, 0].contiguous(), None),
        "form2": (6, seq[3].contiguous(), POSTURE_SEQ_SHARED),
        "form3": (6, seq, POSTURE_SEQ_BATCHED),
        "form3b": (6, seq_b, POSTURE_SEQ_BATCHED),
        "form3_T4": (4, seq[:, :4].contiguous(), POSTURE_SEQ_BATCHED),
    }
    bufs = {T: (q0.clone(), torch.empty((B, T, nq), device="cuda:0"), torch.empty((B, T), dtype=torch.int32, device="cuda:0"),
                torch.empty((B, T), dtype=torch.int32, device="cuda:0")) for T in fts}

    def run(prob, k):
        T, pt, form = calls[k]
        q, qt, it, st = bufs[T]
        q.copy_(q0); qt.fill_(float("nan")); it.fill_(-1); st.fill_(-1)
        inp, keep, _, _ = prob._inputs(None, fts[T], pt, None, dtype=torch.float32)
        if form is not None:
            inp.posture_batched = form
        _lib.check(prob.lib.bik_track(prob.handle, B, T, q.data_ptr(), C.byref(inp), None, c["kw"]["dt"], c["kw"]["damping"],
                                      CONV["max_iters"], CONV["pos_threshold"], CONV["ori_threshold"], 1, qt.data_ptr(), it.data_ptr(),
                                      st.data_ptr(), None, _stream()))
        return q.clone(), qt.clone(), it.clone(), st.clone()

    fresh = {k: run(Problem(c["model"], c["spec"]), k) for k in calls}
    for k in ["form0", "form3", "form3", "form1", "form2", "form2", "form3b", "form3", "form3_T4", "form3_T4", "form2", "form0",
              "form3b", "form1"]:
        for x, y in zip(run(c["prob"], k), fresh[k]):
            _equal(x, y)


def test_sequence_forms_rejected_outside_track():
    """posture_batched = 2 or 3 is refused with BIK_ERR_INVALID by every entry point that is not a bik_track one (bik_solve and
    the other dense entry points take no bik_inputs)."""
    from mink_b200._abi import POSTURE_SEQ_BATCHED, POSTURE_SEQ_SHARED

    c = _gpu_case("ur5e", np.float32, B=8, T=2, seed=1)
    prob, lib, B, nq, nv, K = c["prob"], c["prob"].lib, 8, c["fm"].nq, c["fm"].nv, c["spec"].nrows
    for dtype in (torch.float32, torch.float64):
        z = lambda *s: torch.zeros(s, dtype=dtype, device="cuda:0")
        q, dq, J, e, ep = z(B, nq), z(B, nv), z(B, K, nv), z(B, K), z(B, 1, nv)
        w = torch.ones((B, K), dtype=dtype, device="cuda:0")
        it, st = torch.zeros(B, dtype=torch.int32, device="cuda:0"), torch.zeros(B, dtype=torch.int32, device="cuda:0")
        f64 = dtype == torch.float64
        sfx = "64" if f64 else ""
        for form in (POSTURE_SEQ_SHARED, POSTURE_SEQ_BATCHED):
            inp, keep, _, _ = prob._inputs(None, c["d"]["ft"][:, 0].to(dtype), z(B, 2, 1, nq), None, dtype=dtype)
            inp.posture_batched = form
            r = C.byref(inp)
            conv = (1e-2, 1e-3, 5, 1e-3, 1e-3, 1, it.data_ptr(), st.data_ptr(), None)
            calls = {
                "bik_step": lambda: getattr(lib, "bik_step" + sfx)(prob.handle, B, q.data_ptr(), r, 1e-2, 1e-3, 1, 1, dq.data_ptr(), st.data_ptr(), None),
                "bik_step_weighted": lambda: getattr(lib, "bik_step_weighted" + sfx)(prob.handle, B, q.data_ptr(), r, w.data_ptr(), 1e-2, 1e-3, 1, 1,
                                                                                   dq.data_ptr(), st.data_ptr(), None),
                "bik_converge": lambda: getattr(lib, "bik_converge" + sfx)(prob.handle, B, q.data_ptr(), r, *conv),
                "bik_converge_weighted": lambda: getattr(lib, "bik_converge_weighted" + sfx)(prob.handle, B, q.data_ptr(), r, w.data_ptr(), *conv),
                "bik_fk_jac": lambda: getattr(lib, "bik_fk_jac" + sfx)(prob.handle, B, r, 1e-2, J.data_ptr(), e.data_ptr(), ep.data_ptr(), None, None, None),
            }
            for fn, call in calls.items():
                rc = call()
                assert rc == -1, (fn + sfx, form, rc)
                assert "bik_track" in lib.bik_last_error().decode(), fn
            if not f64:   # bik_step_host: host buffers, fp32 only
                qh, fth = np.zeros((B, nq), np.float32), np.ascontiguousarray(c["ft"][:, 0], np.float32)
                pth = np.zeros((2, 1, nq), np.float32)
                hin = type(inp)()
                hin.frame_targets, hin.posture_targets, hin.posture_batched = fth.ctypes.data, pth.ctypes.data, form
                dqh, sth = np.zeros((B, nv), np.float32), np.zeros(B, np.int32)
                rc = lib.bik_step_host(prob.handle, B, qh.ctypes.data, C.byref(hin), 1e-2, 1e-3, 1, 1, dqh.ctypes.data, sth.ctypes.data, None, None)
                assert rc == -1 and "bik_track" in lib.bik_last_error().decode()


def _g1_api(B, T, seed=7):
    import mink_b200 as mink

    c = _gpu_case("g1", np.float32, B=B, T=T, seed=seed)
    wl, fm = WORKLOADS["g1"], c["fm"]

    def setup(q0, posture):
        cfg = mink.Configuration(fm, q0)
        tasks = [mink.FrameTask(f["name"], f["type"], f["position_cost"], f["orientation_cost"], lm_damping=f["lm_damping"])
                 for f in wl["frames"]]
        post = mink.PostureTask(fm, cost=wl["posture"]["cost"])
        post.set_target(posture)
        limits = [mink.ConfigurationLimit(fm),
                  mink.VelocityLimit(fm, {n: np.pi for n, t in zip(fm.names["joint"], fm.node_type) if t >= 2})]
        pelvis = cfg.get_transform_frame_to_world(wl["frames"][2]["name"], wl["frames"][2]["type"])
        tasks[2].set_target(pelvis)   # held for every frame
        return cfg, tasks + [post], limits

    return c, setup, mink


def test_track_ik_posture_sequence_equals_converge_ik():
    """G1: foot sequences, a held pelvis target and a PostureTask following a joint-space sequence.  track_ik == converge_ik
    after posture_task.set_target(seq[t]) on every frame, for a float32 batch ([B, T, nq] CUDA tensor) and for a single fp64
    configuration ([T, nq] numpy array)."""
    from mink_b200.lie import SE3

    c, setup, mink = _g1_api(B=64, T=5)
    ft = c["ft"].astype(np.float64)
    pseq = c["pseq"][:, :, 0]                       # [B, T, nq]
    dt, damping = c["kw"]["dt"], c["kw"]["damping"]
    q0 = torch.tensor(c["q0"], dtype=torch.float32, device="cuda:0")

    cfg, tasks, limits = setup(q0.clone(), c["q0"].astype(np.float64))
    targets = {tasks[0]: c["d"]["ft"][:, :, 0], tasks[1]: SE3(ft[:, :, 1]), tasks[3]: torch.tensor(pseq, device="cuda:0")}
    q_traj, iters, ok = mink.track_ik(cfg, tasks, dt, targets, damping=damping, limits=limits, **CONV)
    cfg2, tasks2, limits2 = setup(q0.clone(), c["q0"].astype(np.float64))
    for t in range(c["T"]):
        tasks2[0].set_target(SE3(ft[:, t, 0]))
        tasks2[1].set_target(SE3(ft[:, t, 1]))
        tasks2[3].set_target(pseq[:, t].astype(np.float64))
        it, okt = mink.converge_ik(cfg2, tasks2, dt, damping=damping, limits=limits2, **CONV)
        _equal(q_traj[:, t], cfg2.q_device)
        np.testing.assert_array_equal(iters[:, t].cpu().numpy(), it)
        np.testing.assert_array_equal(ok[:, t].cpu().numpy(), okt)

    one, tasks1, limits1 = setup(c["q0"][0].astype(np.float64), c["q0"][0].astype(np.float64))
    q1, it1, ok1 = mink.track_ik(one, tasks1, dt, {tasks1[0]: ft[0, :, 0], tasks1[1]: ft[0, :, 1], tasks1[3]: pseq[0].astype(np.float64)},
                                 damping=damping, limits=limits1, **CONV)
    two, tasks2, limits2 = setup(c["q0"][0].astype(np.float64), c["q0"][0].astype(np.float64))
    for t in range(c["T"]):
        tasks2[0].set_target(SE3(ft[0, t, 0]))
        tasks2[1].set_target(SE3(ft[0, t, 1]))
        tasks2[3].set_target(pseq[0, t].astype(np.float64))
        it, okt = mink.converge_ik(two, tasks2, dt, damping=damping, limits=limits2, **CONV)
        np.testing.assert_array_equal(q1[t], two.q)
        assert it1[t] == it and ok1[t] == okt


def test_track_ik_posture_sequence_errors():
    c, setup, mink = _g1_api(B=8, T=3)
    ft, fm = c["ft"].astype(np.float64), c["fm"]
    cfg, tasks, limits = setup(torch.tensor(c["q0"], dtype=torch.float32, device="cuda:0"), c["q0"].astype(np.float64))
    feet = {tasks[0]: ft[:, :, 0], tasks[1]: ft[:, :, 1]}
    damp = mink.DampingTask(fm, cost=0.1)
    with pytest.raises(mink.InvalidTarget):   # a DampingTask's target is qpos0
        mink.track_ik(cfg, tasks + [damp], 1e-2, {**feet, damp: np.zeros((3, fm.nq))}, limits=limits)
    with pytest.raises(mink.InvalidTarget):   # not [T, nq] / [B, T, nq]
        mink.track_ik(cfg, tasks, 1e-2, {**feet, tasks[3]: np.zeros((3, fm.nq - 1))}, limits=limits)
    with pytest.raises(mink.InvalidTarget):   # another number of frames than the other sequences
        mink.track_ik(cfg, tasks, 1e-2, {**feet, tasks[3]: np.zeros((4, fm.nq))}, limits=limits)
