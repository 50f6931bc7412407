"""The cost of a posture target sequence in bik_track (needs a GPU).

  python tools/bench_track_posture.py [--B 4096,65536] [--T 100] [--reps 5]

G1 with the headline tasks and limits (workload "g1"), T frames of the seeded smooth trajectory of tools/bench_track.py: frame
targets are the CUDA FK of q0 (+) (t+1)/T delta, delta ~ N(0, 0.3^2) on the hinge dofs; max_iters 10, thresholds 1e-3.  Three
cases, alternating in one process:
  (a) held:     each instance's posture target is its q0, one target for the whole call (posture_batched = 1);
  (b) repeated: the same target repeated as a [B, T, P, nq] sequence (posture_batched = 3).  Its outputs must equal (a)'s bit
                for bit, so the difference in time is the per-frame copy of the posture rows alone;
  (c) path:     the joint path q0 (+) (t+1)/T delta itself as the sequence, as a retargeting pipeline would pass it.
Prints one JSON line per batch size: wall time per call (CUDA events; median and all repetitions), the overhead of (b) and (c)
over (a), the pass counts, whether (b) equals (a), the card and its power limit.
"""
import argparse
import json
import os
import subprocess
import sys

import numpy as np
import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
from mink_b200._abi import spec_from_workload  # noqa: E402
from mink_b200.engine import DeviceModel, Problem  # noqa: E402
from mink_b200.workloads import WORKLOADS, load_flat, make_inputs, task_frames  # noqa: E402

CONV = dict(max_iters=10, pos_threshold=1e-3, ori_threshold=1e-3)


def card():
    try:
        out = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader", "-i", "0"],
                             capture_output=True, text=True, timeout=30).stdout.strip()
    except (OSError, subprocess.TimeoutExpired):
        out = ""
    return out or torch.cuda.get_device_name(0)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--B", default="4096,65536")
    ap.add_argument("--T", type=int, default=100)
    ap.add_argument("--reps", type=int, default=5)
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("bench_track_posture.py needs a CUDA device")
    wl = WORKLOADS["g1"]
    fm = load_flat(wl["robot"])
    spec = spec_from_workload(fm, wl)
    model = DeviceModel(fm, 0)
    prob = Problem(model, spec)
    frames = task_frames(wl, fm)
    dev = "cuda:0"
    gpu = card()

    def fk(qq):
        p, _ = model.fk(qq, frames)
        return p.cpu().numpy().astype(np.float64), None

    T = args.T
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
        path = torch.empty((B, T, 1, fm.nq), device=dev, dtype=torch.float32)
        for t in range(T):
            path[:, t, 0] = q0 + frac[t] * delta
            poses, _ = model.fk(path[:, t, 0], frames)
            ft[:, t] = poses
        held = q0[:, None, :].clone()
        cases = {"held": (held, False), "repeated": (held[:, None].expand(B, T, 1, fm.nq).contiguous(), True), "path": (path, True)}
        kw = dict(dt=wl["dt"], damping=wl["damping"], **CONV)
        ev = [torch.cuda.Event(enable_timing=True) for _ in range(2)]

        def run(k):
            pt, is_seq = cases[k]
            q = q0.clone()
            ev[0].record()
            q_traj, it, st, passes = prob.track(q, ft, pt, None, posture_seq=is_seq, **kw)
            ev[1].record()
            torch.cuda.synchronize()
            return ev[0].elapsed_time(ev[1]), (q_traj, it, st, q), int(passes)

        for k in cases:   # warm-up: graphs, launch geometry, workspace
            run(k)
        ms = {k: [] for k in cases}
        for r in range(args.reps):
            out = {k: run(k) for k in cases}
            for k in cases:
                ms[k].append(out[k][0])
            if r == 0:
                identical = all(torch.equal(x, y) for x, y in zip(out["held"][1], out["repeated"][1]))
                passes = {k: out[k][2] for k in cases}
                iters = {k: int(out[k][1][1].sum()) for k in cases}
            del out
        med = {k: float(np.median(v)) for k, v in ms.items()}
        print(json.dumps({
            "workload": "g1", "B": B, "T": T, **CONV, "card": gpu, "repeated_identical_to_held": identical,
            "ms": {k: round(v, 3) for k, v in med.items()}, "ms_all": {k: [round(x, 3) for x in v] for k, v in ms.items()},
            "overhead_pct": {k: round(100.0 * (med[k] / med["held"] - 1.0), 2) for k in ("repeated", "path")},
            "passes": passes, "iters_total": iters,
        }), flush=True)
        del ft, path, cases


if __name__ == "__main__":
    main()
