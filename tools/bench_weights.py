"""What per-instance task weights cost (needs a GPU).

  python tools/bench_weights.py [--B 65536] [--steps 200] [--T 100] [--reps 5]

G1 with the headline tasks and limits (workload "g1", K = 18 weighted rows) at B instances, fp32, in one process:

  step   bik_step against bik_step_weighted, one call per step, `steps` calls per timed window (CUDA events), the variants
         alternating window by window: no weights, all-ones weights (the same QPs: what reading and applying the weights
         costs) and random weights in [0, 1] (other QPs, so K2's active-set work differs too).
  track  the bik_track workload of tools/bench_track.py (T frames of a seeded smooth trajectory, max_iters 10, thresholds
         1e-3) without weights, with all-ones [B][T][K] weights and with random ones, alternating call by call.

The all-ones variants must give the unweighted outputs bit for bit; the script checks that.  Prints one JSON line per part:
median times, every repetition, the overhead of the all-ones variant over the unweighted one, the card and its power limit.
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
    ap.add_argument("--B", type=int, default=65536)
    ap.add_argument("--steps", type=int, default=200)
    ap.add_argument("--T", type=int, default=100)
    ap.add_argument("--reps", type=int, default=5)
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("bench_weights.py needs a CUDA device")
    wl = WORKLOADS["g1"]
    fm = load_flat(wl["robot"])
    spec = spec_from_workload(fm, wl)
    model = DeviceModel(fm, 0)
    prob = Problem(model, spec)
    frames = task_frames(wl, fm)
    dev, B, T, K = "cuda:0", args.B, args.T, prob.K
    gpu = card()
    ev = [torch.cuda.Event(enable_timing=True) for _ in range(2)]

    def fk(qq):
        p, _ = model.fk(qq, frames)
        return p.cpu().numpy().astype(np.float64), None

    inp = make_inputs(fm, wl, B, fk, seed=7)
    q0 = torch.tensor(inp["q"], dtype=torch.float32, device=dev)
    ft0 = torch.tensor(inp["frame_targets"], dtype=torch.float32, device=dev)
    pt = torch.tensor(inp["posture_target"], dtype=torch.float32, device=dev)
    gen = torch.Generator(device=dev).manual_seed(9)
    weights = {"none": None, "ones": torch.ones((B, K), device=dev), "random": torch.rand((B, K), device=dev, generator=gen)}

    # ---- step ----------------------------------------------------------------------------------------------------------
    dq = torch.empty((B, fm.nv), device=dev)
    st = torch.empty(B, device=dev, dtype=torch.int32)
    skw = dict(dt=wl["dt"], damping=wl["damping"], dq=dq, status=st)
    outs = {}
    for name, w in weights.items():   # warm-up, and the outputs of one step from q0
        prob.step(q0.clone(), ft0, pt, None, weights=w, **skw)
        torch.cuda.synchronize()
        outs[name] = (dq.clone(), st.clone())
    identical_step = bool(torch.equal(outs["ones"][0], outs["none"][0]) and torch.equal(outs["ones"][1], outs["none"][1]))
    times = {n: [] for n in weights}
    q = q0.clone()
    for _ in range(args.reps):
        for name, w in weights.items():
            ev[0].record()
            for _ in range(args.steps):
                prob.step(q, ft0, pt, None, weights=w, **skw)
            ev[1].record()
            torch.cuda.synchronize()
            times[name].append(ev[0].elapsed_time(ev[1]) / args.steps)
    med = {n: float(np.median(v)) for n, v in times.items()}
    print(json.dumps({
        "part": "step", "workload": "g1", "B": B, "K": K, "steps_per_window": args.steps, "card": gpu, "identical_outputs": identical_step,
        "ms_per_step": {n: round(v, 4) for n, v in med.items()}, "ms_per_step_all": {n: [round(x, 4) for x in v] for n, v in times.items()},
        "overhead_ones_pct": round(100 * (med["ones"] / med["none"] - 1), 2), "overhead_random_pct": round(100 * (med["random"] / med["none"] - 1), 2),
        "weights_bytes_per_step": B * K * 4,
    }), flush=True)

    # ---- track (the workload of tools/bench_track.py) ---------------------------------------------------------------------
    rng = np.random.default_rng(8)
    delta = torch.zeros_like(q0)
    for n in range(fm.nnode):
        if int(fm.node_type[n]) >= 2:
            delta[:, int(fm.node_qadr[n])] = torch.tensor(rng.normal(0.0, 0.3, size=B), dtype=torch.float32, device=dev)
    frac = torch.arange(1, T + 1, device=dev, dtype=torch.float32) / T
    ft = torch.empty((B, T, len(frames), 7), device=dev)
    for t in range(T):
        ft[:, t], _ = model.fk(q0 + frac[t] * delta, frames)
    ptt = q0[:, None, :].clone()
    tweights = {"none": None, "ones": torch.ones((B, T, K), device=dev), "random": torch.rand((B, T, K), device=dev, generator=gen)}
    del weights
    tkw = dict(dt=wl["dt"], damping=wl["damping"], **CONV)

    def run_track(w):
        q = q0.clone()
        ev[0].record()
        q_traj, it, st_, passes = prob.track(q, ft, ptt, None, weights=w, **tkw)
        ev[1].record()
        torch.cuda.synchronize()
        return ev[0].elapsed_time(ev[1]), q_traj, it, st_, int(passes)

    first = {n: run_track(w) for n, w in tweights.items()}   # warm-up (graphs, workspace) and the outputs
    identical_track = all(torch.equal(a, b) for a, b in zip(first["ones"][1:4], first["none"][1:4]))
    ttimes = {n: [] for n in tweights}
    passes = {n: first[n][4] for n in tweights}
    for _ in range(args.reps):
        for name, w in tweights.items():
            ttimes[name].append(run_track(w)[0])
    tmed = {n: float(np.median(v)) for n, v in ttimes.items()}
    print(json.dumps({
        "part": "track", "workload": "g1", "B": B, "T": T, "K": K, **CONV, "card": gpu, "identical_outputs": identical_track,
        "track_ms": {n: round(v, 2) for n, v in tmed.items()}, "track_ms_all": {n: [round(x, 2) for x in v] for n, v in ttimes.items()},
        "passes": passes, "ms_per_pass": {n: round(tmed[n] / passes[n], 4) for n in tmed},
        "overhead_ones_pct": round(100 * (tmed["ones"] / tmed["none"] - 1), 2),
    }), flush=True)


if __name__ == "__main__":
    main()
