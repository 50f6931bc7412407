"""Small invocations of every kernel path for compute-sanitizer (memcheck / racecheck): K1 packed and dense (direct + staged),
K1 fp64, both K2 paths (small-group 32/64-bit masks, general with collision rows), fp64 entry points, bik_converge, bik_track and
bik_converge64 / bik_track64 (host-polled, also with posture target sequences), bik_step_host.
Ragged batches so that tail tiles run.  Usage:  compute-sanitizer --tool racecheck python tools/sanitize_run.py"""
import os
import sys

import numpy as np
import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
from mink_b200._abi import spec_from_workload
from mink_b200.engine import DeviceModel, Problem
from mink_b200.workloads import WORKLOADS, load_flat

GOLD = os.path.join(os.path.dirname(os.path.dirname(os.path.abspath(__file__))), "tests", "golden")
for name, env in (("g1", {}), ("g1", {"BIK_K2_PATH": "dense"}), ("g1", {"BIK_USE_TMA": "0"}), ("shadow", {}), ("spot", {}), ("edge", {}),
                  ("g1_full", {}), ("g1_rel", {}), ("ur5e_dls", {}), ("ur5e_damp", {}), ("ur5e_wall", {})):
    os.environ.update(env)
    wl = WORKLOADS[name]
    fm = load_flat(wl["robot"])
    spec = spec_from_workload(fm, wl)
    g = dict(np.load(os.path.join(GOLD, name + ".npz")))
    model = DeviceModel(fm, 0)
    prob = Problem(model, spec)
    rep = -(-45 // g["q"].shape[0])
    tile = lambda a: None if a is None else np.tile(a, (rep,) + (1,) * (a.ndim - 1))[:45]
    q0, ft, ct = tile(g["q"]), tile(g["frame_targets"]), tile(g.get("com_target"))
    pt = g["posture_target"]
    dt, damping = float(g["dt"]), float(g["damping"])
    for dtype in (torch.float32, torch.float64):
        q = torch.tensor(q0, dtype=dtype, device="cuda:0")
        J, e, ep, Gc, hc = prob.fk_jac(q, ft, pt, ct, dt=dt)                      # K1 dense
        prob.solve(q, J, e, ep, Gc, hc, dt, damping)                              # K2 on dense rows
        dq, st = prob.step(q, ft, pt, ct, dt=dt, damping=damping, nsteps=3, integrate=True)   # K1 packed + K2 fused integrate, warm-started
        assert int((st & ~1).max()) == 0, (name, env, dtype, st)
    q = torch.tensor(q0, dtype=torch.float32, device="cuda:0")
    prob.converge(q, ft, pt, ct, dt=dt, damping=damping, max_iters=4, pos_threshold=2e-3, ori_threshold=2e-3)
    # track: 3 frames (the same targets, moved by frame index), ragged lengths, the host-polled loop
    seq = lambda a: None if a is None else np.stack([a, a, a], axis=1)
    fts = seq(ft)
    if fts is not None:
        fts[:, 1:, :, 4:] += 1e-3 * np.arange(1, 3)[None, :, None, None]
    os.environ["BIK_CONVERGE_GRAPH"] = "0"
    prob.track(q, fts, pt, seq(ct), lengths=torch.arange(45, device="cuda:0", dtype=torch.int32) % 4, dt=dt, damping=damping,
               max_iters=4, pos_threshold=2e-3, ori_threshold=2e-3, check_every=2)
    q64 = torch.tensor(q0, dtype=torch.float64, device="cuda:0")   # the fp64 loops, host-polled
    prob.converge(q64, ft, pt, ct, dt=dt, damping=damping, max_iters=4, pos_threshold=2e-3, ori_threshold=2e-3, check_every=2)
    prob.track(q64, fts, pt, seq(ct), lengths=torch.arange(45, device="cuda:0", dtype=torch.int32) % 4, dt=dt, damping=damping,
               max_iters=4, pos_threshold=2e-3, ori_threshold=2e-3, check_every=2)
    if spec.nposture:   # posture target sequences: per instance (fp32, K1 copies each frame's rows) and shared (fp64)
        pts = np.broadcast_to(np.asarray(pt, np.float64).reshape(1, 1, spec.nposture, fm.nq), (45, 3, spec.nposture, fm.nq)).copy()
        pts[:, 1:] += 1e-3 * np.arange(1, 3)[None, :, None, None]
        prob.track(q, fts, pts, seq(ct), lengths=torch.arange(45, device="cuda:0", dtype=torch.int32) % 4, dt=dt, damping=damping,
                   max_iters=4, pos_threshold=2e-3, ori_threshold=2e-3, check_every=2, posture_seq=True)
        prob.track(q64, fts, pts[0], seq(ct), dt=dt, damping=damping, max_iters=4, pos_threshold=2e-3, ori_threshold=2e-3,
                   check_every=2, posture_seq=True)
    os.environ.pop("BIK_CONVERGE_GRAPH")
    prob.step_host(q0.astype(np.float32), ft, pt, ct, dt=dt, damping=damping, nsteps=1, integrate=True)
    torch.cuda.synchronize()
    print("ok", name, env, prob.describe(damping), flush=True)
    prob.close()
    for k in env:
        os.environ.pop(k)
print("done")
