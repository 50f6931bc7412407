"""Held targets in bik_track (bik_track_hold) against the calls they replace (needs a GPU).

  python tools/bench_track_hold.py [--B 4096,65536] [--T 100] [--reps 3] [--run 10]

G1 with the headline tasks and limits (workload "g1") and the trajectory of tools/bench_track.py: T frames, targets the CUDA FK
of q0 (+) (t+1)/T delta, max_iters 10, thresholds 1e-3, fp32.  In one process, alternating:

  track      bik_track (no hold mask; what bik_track_coll runs without collision arguments)
  zero_mask  bik_track_hold with an all-zero [B, T, H] mask: the cost of the hold kernel and of reading the mask
  hold       the two feet held in alternating `--run`-frame runs (left on runs 0, 2, ..., right on runs 1, 3, ...)
  split      what a caller does without held targets: the sequence split at every run boundary, and at each boundary
             bik_fk of the configuration reached so far, the held foot's targets set to its pose, one bik_track call

The first repetition compares outputs: track against zero_mask (identical expected), hold against split (q_traj max
difference, iters and status agreement).  Prints one JSON line per batch size with the wall times (CUDA events), the card
and its power limit read in the same process.
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
from mink_b200.workloads import WORKLOADS, load_flat, make_inputs, task_frames  # noqa: E402


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--B", default="4096,65536")
    ap.add_argument("--T", type=int, default=100)
    ap.add_argument("--reps", type=int, default=3)
    ap.add_argument("--run", type=int, default=10, help="frames per hold run")
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("bench_track_hold.py needs a CUDA device")
    wl = WORKLOADS["g1"]
    fm = load_flat(wl["robot"])
    spec = spec_from_workload(fm, wl)
    model = DeviceModel(fm, 0)
    prob = Problem(model, spec)
    frames = task_frames(wl, fm)   # left foot, right foot, pelvis
    H = spec.nframe + spec.ncom + spec.nposture
    dev, T, R = "cuda:0", args.T, args.run
    gpu = card()

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
        pt = q0[:, None, :].clone()
        kw = dict(dt=wl["dt"], damping=wl["damping"], **CONV)
        zero = torch.zeros((B, T, H), device=dev, dtype=torch.uint8)
        feet = torch.zeros_like(zero)
        run_of = torch.arange(T, device=dev) // R
        feet[:, :, 0] = (run_of % 2 == 0).to(torch.uint8)
        feet[:, :, 1] = (run_of % 2 == 1).to(torch.uint8)
        ev = [torch.cuda.Event(enable_timing=True) for _ in range(2)]

        def timed(fn):
            ev[0].record()
            out = fn()
            ev[1].record()
            torch.cuda.synchronize()
            return ev[0].elapsed_time(ev[1]), out

        def run_track(hold=None):
            q = q0.clone()
            return timed(lambda: prob.track(q, ft, pt, None, hold=hold, **kw)[:3])

        def run_split():
            def body():
                q = q0.clone()
                q_traj = torch.empty((B, T, fm.nq), device=dev, dtype=torch.float32)
                its = torch.empty((B, T), device=dev, dtype=torch.int32)
                sts = torch.empty_like(its)
                for t0 in range(0, T, R):
                    t1 = min(T, t0 + R)
                    f = (t0 // R) % 2   # the foot held on this run
                    seg = ft[:, t0:t1].clone()
                    seg[:, :, f] = model.fk(q, [frames[f]])[0][:, None, 0]
                    q_traj[:, t0:t1], its[:, t0:t1], sts[:, t0:t1], _ = prob.track(q, seg.contiguous(), pt, None, **kw)
                return q_traj, its, sts
            return timed(body)

        runs = {"track": run_track, "zero_mask": lambda: run_track(zero), "hold": lambda: run_track(feet), "split": run_split}
        for f in runs.values():   # warm-up: graphs, launch geometry, workspace
            f()
        ms = {k: [] for k in runs}
        cmp = {}
        for r in range(args.reps):
            outs = {}
            for k, f in runs.items():
                t, outs[k] = f()
                ms[k].append(t)
            if r == 0:
                cmp["zero_mask_identical_to_track"] = all(torch.equal(a, b) for a, b in zip(outs["track"], outs["zero_mask"]))
                (qa, ia, sa), (qb, ib, sb) = outs["hold"], outs["split"]
                cmp["hold_vs_split"] = {"q_traj_max_abs_diff": float((qa - qb).abs().max()), "identical": bool(torch.equal(qa, qb)),
                                        "iters_equal_fraction": float((ia == ib).float().mean()),
                                        "status_equal_fraction": float((sa == sb).float().mean())}
        med = {k: round(float(np.median(v)), 2) for k, v in ms.items()}
        print(json.dumps({
            "workload": "g1", "precision": "f32", "B": B, "T": T, "run": R, **CONV, "card": gpu,
            "ms": med, "ms_all": {k: [round(x, 2) for x in v] for k, v in ms.items()},
            "zero_mask_over_track": round(med["zero_mask"] / med["track"], 4), "split_over_hold": round(med["split"] / med["hold"], 4),
            **cmp,
        }), flush=True)
        del ft, zero, feet


if __name__ == "__main__":
    main()
