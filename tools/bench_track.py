"""bik_track against the per-frame bik_converge loop it replaces (needs a GPU).

  python tools/bench_track.py [--B 4096,65536] [--T 100] [--reps 3] [--f64]

G1 with the headline tasks and limits (workload "g1"), T frames of a seeded smooth trajectory per instance: targets are the
CUDA FK of q0 (+) (t+1)/T delta, delta ~ N(0, 0.3^2) on the hinge dofs, each instance's posture target its q0; max_iters 10,
thresholds 1e-3.  In one process, alternating: one bik_track call, and T bik_converge calls on the same inputs (the examples'
outer loop, one host round trip per frame).  The first repetition checks that both give identical q_traj, iters and status.
Prints one JSON line per batch size: wall time per call (CUDA events), frames/s (B*T / wall), IK steps/s (sum of iters /
wall), the pass counts (bik_track: max_b sum_t (iters + 1); per-frame loop: sum_t max_b (iters + 1)), the card and its power
limit.

--f64: the same on fp64 buffers, bik_track64 against T bik_converge64 calls, and in the same process fp32 bik_track on the
same inputs rounded to fp32 (the price of fp64: "track32_ms").  The targets are the fp64 FK of the same joint path.
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
    ap.add_argument("--reps", type=int, default=3)
    ap.add_argument("--f64", action="store_true", help="bik_track64 / bik_converge64, with fp32 bik_track for comparison")
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("bench_track.py needs a CUDA device")
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
    dtype = torch.float64 if args.f64 else torch.float32
    for B in (int(b) for b in args.B.split(",")):
        inp = make_inputs(fm, wl, B, fk, seed=7)
        rng = np.random.default_rng(8)
        q0 = torch.tensor(inp["q"], dtype=dtype, device=dev)
        delta = torch.zeros_like(q0)
        for n in range(fm.nnode):
            if int(fm.node_type[n]) >= 2:
                delta[:, int(fm.node_qadr[n])] = torch.tensor(rng.normal(0.0, 0.3, size=B), dtype=dtype, device=dev)
        frac = torch.arange(1, T + 1, device=dev, dtype=dtype) / T
        ft = torch.empty((B, T, len(frames), 7), device=dev, dtype=dtype)
        for t in range(T):
            poses, _ = model.fk(q0 + frac[t] * delta, frames)
            ft[:, t] = poses
        pt = q0[:, None, :].clone()
        kw = dict(dt=wl["dt"], damping=wl["damping"], **CONV)
        ev = [torch.cuda.Event(enable_timing=True) for _ in range(2)]

        def run_track(q0=q0, ft=ft, pt=pt):
            q = q0.clone()
            ev[0].record()
            q_traj, it, st, passes = prob.track(q, ft, pt, None, **kw)
            ev[1].record()
            torch.cuda.synchronize()
            return ev[0].elapsed_time(ev[1]), q_traj, it, st, int(passes)

        def run_loop():
            q = q0.clone()
            q_traj = torch.empty((B, T, fm.nq), device=dev, dtype=dtype)
            its = torch.empty((B, T), device=dev, dtype=torch.int32)
            sts = torch.empty((B, T), device=dev, dtype=torch.int32)
            ev[0].record()
            for t in range(T):
                it, st = prob.converge(q, ft[:, t], pt, None, **kw)
                int(st[0])   # the examples read the result back on every frame
                q_traj[:, t] = q
                its[:, t] = it
                sts[:, t] = st
            ev[1].record()
            torch.cuda.synchronize()
            return ev[0].elapsed_time(ev[1]), q_traj, its, sts

        f32 = (q0.float(), ft.float(), pt.float()) if args.f64 else None
        run_track(); run_loop()   # warm-up: graphs, launch geometry, workspace
        if f32:
            run_track(*f32)
        tt, tl, t32 = [], [], []
        for r in range(args.reps):
            ms_t, qa, ia, sa, passes = run_track()
            ms_l, qb, ib, sb = run_loop()
            if f32:
                t32.append(run_track(*f32)[0])
            if r == 0:
                identical = bool(torch.equal(qa, qb) and torch.equal(ia, ib) and torch.equal(sa, sb))
                steps = int(ia.sum())
                barrier = int((ia + 1).max(0).values.sum())
            tt.append(ms_t); tl.append(ms_l)
        mt, ml = float(np.median(tt)), float(np.median(tl))
        extra = {"track32_ms": round(float(np.median(t32)), 2), "track32_ms_all": [round(x, 2) for x in t32]} if f32 else {}
        print(json.dumps({
            "workload": "g1", "precision": "f64" if args.f64 else "f32", "B": B, "T": T, **CONV, "card": gpu, "identical_outputs": identical,
            "track_ms": round(mt, 2), "loop_ms": round(ml, 2), "track_ms_all": [round(x, 2) for x in tt], "loop_ms_all": [round(x, 2) for x in tl],
            "frames_per_s": {"track": round(B * T / mt * 1e3), "loop": round(B * T / ml * 1e3)},
            "ik_steps_per_s": {"track": round(steps / mt * 1e3), "loop": round(steps / ml * 1e3)},
            "passes": {"track": passes, "per_frame_loop": barrier}, "iters_total": steps, **extra,
        }), flush=True)
        del ft, f32


if __name__ == "__main__":
    main()
