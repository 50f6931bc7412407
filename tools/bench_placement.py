"""Per-instance frame placement (bik_step_placed, bik_track_placed) against the calls without one (needs a GPU).

  python tools/bench_placement.py [--B 4096,65536] [--T 100] [--steps 50] [--reps 5]

G1 with the headline tasks and limits (workload "g1"), fp32.  In one process, alternating:

  step         --steps bik_step calls of one step each, integrating q (no placement: what bik_step_coll runs with NULL)
  step_placed  the same through bik_step_placed, with rows equal to the problem's own placement of every frame task
  track        bik_track over the trajectory of tools/bench_track.py (T frames, max_iters 10, thresholds 1e-3)
  track_placed the same through bik_track_placed with the problem's own placement

Every repetition checks that each pair gives identical outputs (dq / q / status, q_traj / iters / status).  Prints one JSON
line per batch size with the median wall times (CUDA events), the cost of the placed form, and the card and its power limit
read in the same process.
"""
import argparse
import json
import os
import sys

import numpy as np
import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
from bench_track import CONV, card  # noqa: E402
from mink_b200._abi import spec_from_workload  # noqa: E402
from mink_b200.engine import DeviceModel, Problem  # noqa: E402
from mink_b200.ik import _frame_row  # noqa: E402
from mink_b200.workloads import WORKLOADS, load_flat, make_inputs, task_frames  # noqa: E402


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--B", default="4096,65536")
    ap.add_argument("--T", type=int, default=100)
    ap.add_argument("--steps", type=int, default=50)
    ap.add_argument("--reps", type=int, default=5)
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("bench_placement.py needs a CUDA device")
    wl = WORKLOADS["g1"]
    fm = load_flat(wl["robot"])
    spec = spec_from_workload(fm, wl)
    model = DeviceModel(fm, 0)
    prob = Problem(model, spec)
    frames = task_frames(wl, fm)
    dev, T = "cuda:0", args.T
    gpu = card()
    own = torch.tensor(np.stack([_frame_row(t.frame, np.float32) for t in spec.tasks if t.frame is not None]), device=dev)

    def fk(qq):
        p, _ = model.fk(qq, frames)
        return p.cpu().numpy().astype(np.float64), None

    for B in (int(b) for b in args.B.split(",")):
        inp = make_inputs(fm, wl, B, fk, seed=7)
        rng = np.random.default_rng(8)
        q0 = torch.tensor(inp["q"], dtype=torch.float32, device=dev)
        delta = torch.zeros_like(q0)
        for n in range(fm.nnode):
            if int(fm.node_type[n]) >= 2:
                delta[:, int(fm.node_qadr[n])] = torch.tensor(rng.normal(0.0, 0.3, size=B), dtype=torch.float32, device=dev)
        frac = torch.arange(1, T + 1, device=dev, dtype=torch.float32) / T
        ft = torch.empty((B, T, len(frames), 7), device=dev, dtype=torch.float32)
        for t in range(T):
            ft[:, t] = model.fk(q0 + frac[t] * delta, frames)[0]
        ft0 = ft[:, -1].contiguous()
        pt = q0[:, None, :].clone()
        rows = own.expand(B, -1, -1).contiguous()
        ev = [torch.cuda.Event(enable_timing=True) for _ in range(2)]

        def timed(fn):
            ev[0].record()
            out = fn()
            ev[1].record()
            torch.cuda.synchronize()
            return ev[0].elapsed_time(ev[1]), out

        def run_step(placement=None):
            def body():
                q = q0.clone()
                dq = torch.empty((B, fm.nv), device=dev, dtype=torch.float32)
                st = torch.empty(B, device=dev, dtype=torch.int32)
                for _ in range(args.steps):
                    prob.step(q, ft0, pt, None, dt=wl["dt"], damping=wl["damping"], nsteps=1, integrate=True, dq=dq, status=st,
                              placement=placement)
                return q, dq, st
            return timed(body)

        def run_track(placement=None):
            q = q0.clone()
            return timed(lambda: prob.track(q, ft, pt, None, dt=wl["dt"], damping=wl["damping"], **CONV, placement=placement)[:3])

        runs = {"step": run_step, "step_placed": lambda: run_step(rows), "track": run_track, "track_placed": lambda: run_track(rows)}
        for f in runs.values():   # warm-up: graphs, launch geometry, workspace
            f()
        ms = {k: [] for k in runs}
        identical = {"step": True, "track": True}
        for _ in range(args.reps):
            outs = {}
            for k, f in runs.items():
                t, outs[k] = f()
                ms[k].append(t)
            for k in identical:
                identical[k] = identical[k] and all(torch.equal(a, b) for a, b in zip(outs[k], outs[k + "_placed"]))
        med = {k: round(float(np.median(v)), 3) for k, v in ms.items()}
        print(json.dumps({
            "workload": "g1", "precision": "f32", "B": B, "T": T, "steps": args.steps, **CONV, "card": gpu,
            "ms": med, "ms_all": {k: [round(x, 3) for x in v] for k, v in ms.items()},
            "step_placed_over_step": round(med["step_placed"] / med["step"], 4),
            "track_placed_over_track": round(med["track_placed"] / med["track"], 4),
            "identical": identical,
        }), flush=True)
        del ft


if __name__ == "__main__":
    main()
