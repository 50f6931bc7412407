"""What per-instance posture weights cost (needs a GPU).

  python tools/bench_posture_weights.py [--B 65536] [--steps 200] [--T 50] [--reps 5]

G1 with the headline tasks and limits (workload "g1": one PostureTask, P x nv = 43 weights per instance) at B instances, fp32,
in one process, all-ones task weights throughout:

  step   bik_step_weighted against bik_step_weighted_ex, one call per step, `steps` calls per timed window (CUDA events), the
         variants alternating window by window: no posture weights, all-ones posture weights (the same QPs: what reading and
         applying the weights costs) and random posture weights in [0, 1] (other QPs, so K2's active-set work differs too).
  track  the bik_track workload of tools/bench_track.py (T frames of a seeded smooth trajectory, max_iters 10, thresholds
         1e-3) through bik_track_weighted and bik_track_weighted_ex with all-ones and with random [B][T][P][nv] weights,
         alternating call by call.

The all-ones variants must give the outputs without posture weights bit for bit; the script checks that.  Prints one JSON line
per part: median times, every repetition, the overhead of the all-ones variant, the card and its power limit.
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
    ap.add_argument("--T", type=int, default=50)
    ap.add_argument("--reps", type=int, default=5)
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("bench_posture_weights.py needs a CUDA device")
    wl = WORKLOADS["g1"]
    fm = load_flat(wl["robot"])
    spec = spec_from_workload(fm, wl)
    model = DeviceModel(fm, 0)
    prob = Problem(model, spec)
    frames = task_frames(wl, fm)
    dev, B, T, K, P, nv = "cuda:0", args.B, args.T, prob.K, prob.P, fm.nv
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
    w1 = torch.ones((B, K), device=dev)
    pweights = {"weighted": None, "ex_ones": torch.ones((B, P, nv), device=dev),
                "ex_random": torch.rand((B, P, nv), device=dev, generator=gen)}

    # ---- step ----------------------------------------------------------------------------------------------------------
    dq = torch.empty((B, nv), device=dev)
    st = torch.empty(B, device=dev, dtype=torch.int32)
    skw = dict(dt=wl["dt"], damping=wl["damping"], dq=dq, status=st, weights=w1)
    outs = {}
    for name, pw in pweights.items():   # warm-up, and the outputs of one step from q0
        prob.step(q0.clone(), ft0, pt, None, posture_weights=pw, **skw)
        torch.cuda.synchronize()
        outs[name] = (dq.clone(), st.clone())
    identical_step = all(torch.equal(a, b) for a, b in zip(outs["ex_ones"], outs["weighted"]))
    times = {n: [] for n in pweights}
    q = q0.clone()
    for _ in range(args.reps):
        for name, pw in pweights.items():
            ev[0].record()
            for _ in range(args.steps):
                prob.step(q, ft0, pt, None, posture_weights=pw, **skw)
            ev[1].record()
            torch.cuda.synchronize()
            times[name].append(ev[0].elapsed_time(ev[1]) / args.steps)
    med = {n: float(np.median(v)) for n, v in times.items()}
    print(json.dumps({
        "part": "step", "workload": "g1", "B": B, "P": P, "nv": nv, "steps_per_window": args.steps, "card": gpu,
        "identical_outputs": identical_step, "ms_per_step": {n: round(v, 4) for n, v in med.items()},
        "ms_per_step_all": {n: [round(x, 4) for x in v] for n, v in times.items()},
        "overhead_ones_pct": round(100 * (med["ex_ones"] / med["weighted"] - 1), 2),
        "overhead_random_pct": round(100 * (med["ex_random"] / med["weighted"] - 1), 2),
        "posture_weights_bytes_per_step": B * P * nv * 4,
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
    tw1 = torch.ones((B, T, K), device=dev)
    del pweights
    tpweights = {"weighted": None, "ex_ones": torch.ones((B, T, P, nv), device=dev),
                 "ex_random": torch.rand((B, T, P, nv), device=dev, generator=gen)}
    tkw = dict(dt=wl["dt"], damping=wl["damping"], weights=tw1, **CONV)

    def run_track(pw):
        q = q0.clone()
        ev[0].record()
        q_traj, it, st_, passes = prob.track(q, ft, ptt, None, posture_weights=pw, **tkw)
        ev[1].record()
        torch.cuda.synchronize()
        return ev[0].elapsed_time(ev[1]), q_traj, it, st_, int(passes)

    first = {n: run_track(pw) for n, pw in tpweights.items()}   # warm-up (graphs, workspace) and the outputs
    identical_track = all(torch.equal(a, b) for a, b in zip(first["ex_ones"][1:4], first["weighted"][1:4]))
    ttimes = {n: [] for n in tpweights}
    passes = {n: first[n][4] for n in tpweights}
    for _ in range(args.reps):
        for name, pw in tpweights.items():
            ttimes[name].append(run_track(pw)[0])
    tmed = {n: float(np.median(v)) for n, v in ttimes.items()}
    print(json.dumps({
        "part": "track", "workload": "g1", "B": B, "T": T, "P": P, "nv": nv, **CONV, "card": gpu, "identical_outputs": identical_track,
        "track_ms": {n: round(v, 2) for n, v in tmed.items()}, "track_ms_all": {n: [round(x, 2) for x in v] for n, v in ttimes.items()},
        "passes": passes, "ms_per_pass": {n: round(tmed[n] / passes[n], 4) for n in tmed},
        "overhead_ones_pct": round(100 * (tmed["ex_ones"] / tmed["weighted"] - 1), 2),
    }), flush=True)


if __name__ == "__main__":
    main()
