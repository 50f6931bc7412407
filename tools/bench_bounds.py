"""What per-instance joint limits cost (needs a GPU).

  python tools/bench_bounds.py [--B 65536] [--steps 200] [--T 50] [--reps 5]

G1 with the headline tasks and limits (workload "g1": a ConfigurationLimit and a VelocityLimit, three [B][nv] fp32 bound buffers
with nv = 43) at B instances, fp32, in one process, all-ones task weights throughout:

  step   bik_step_weighted (what bik_step_weighted_ex runs with null posture weights, and bik_step_bounded with null bounds)
         against bik_step_bounded, one call per step, `steps` calls per timed window (CUDA events), the variants alternating
         window by window: no bounds, bounds equal to the problem's (the same QPs: what reading and applying the bounds costs)
         and random narrowing around q0 (other QPs, so K2's active-set work differs too).
  track  the bik_track workload of tools/bench_track.py (T frames of a seeded smooth trajectory, max_iters 10, thresholds
         1e-3) through bik_track_weighted and bik_track_bounded with the problem's and with randomly narrowed bounds,
         alternating call by call.

The variants with the problem's bounds must give the outputs without bounds bit for bit; the script checks that.  Prints one
JSON line per part: median times, every repetition, the overhead of the problem's-bounds variant, the card and its power limit.
"""
import argparse
import json
import os
import subprocess
import sys

import numpy as np
import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
from mink_b200._abi import LIMIT_CONFIGURATION, LIMIT_VELOCITY, spec_from_workload  # noqa: E402
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
        raise SystemExit("bench_bounds.py needs a CUDA device")
    wl = WORKLOADS["g1"]
    fm = load_flat(wl["robot"])
    spec = spec_from_workload(fm, wl)
    model = DeviceModel(fm, 0)
    prob = Problem(model, spec)
    frames = task_frames(wl, fm)
    dev, B, T, K, nv = "cuda:0", args.B, args.T, prob.K, fm.nv
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
    # the problem's bounds per tangent dof, as its image stores them (fp32), and a random narrowing around q0
    lo0, up0, vm0 = (torch.full((nv,), v, device=dev) for v in (-np.inf, np.inf, np.inf))
    for l in spec.limits:
        if l.kind == LIMIT_CONFIGURATION:
            lo0[l.dof] = torch.tensor(np.float32(l.lower), device=dev)
            up0[l.dof] = torch.tensor(np.float32(l.upper), device=dev)
        elif l.kind == LIMIT_VELOCITY:
            vm0[l.dof] = torch.tensor(np.float32(l.vmax), device=dev)
    qd = torch.zeros((B, nv), device=dev)
    qa = torch.as_tensor(fm.dof_qadr, device=dev)
    qd[:, qa >= 0] = q0[:, qa[qa >= 0]]
    qc = torch.minimum(torch.maximum(qd, lo0), up0)
    u = lambda: torch.rand((B, nv), device=dev, generator=gen)
    fin = torch.isfinite(lo0) & torch.isfinite(up0)
    lo_r = torch.where(fin, lo0 + u() * (torch.where(fin, qc - lo0, 0)), lo0)
    up_r = torch.where(fin, qc + u() * (torch.where(fin, up0 - qc, 0)), up0)
    vm_r = torch.where(torch.isfinite(vm0), u() * vm0, vm0)
    bset = {"weighted": None, "bounded_problem": tuple(x.expand(B, nv).contiguous() for x in (lo0, up0, vm0)),
            "bounded_random": (lo_r, up_r, vm_r)}

    # ---- step ----------------------------------------------------------------------------------------------------------
    dq = torch.empty((B, nv), device=dev)
    st = torch.empty(B, device=dev, dtype=torch.int32)
    skw = dict(dt=wl["dt"], damping=wl["damping"], dq=dq, status=st, weights=w1)
    outs = {}
    for name, bd in bset.items():   # warm-up, and the outputs of one step from q0
        prob.step(q0.clone(), ft0, pt, None, bounds=bd, **skw)
        torch.cuda.synchronize()
        outs[name] = (dq.clone(), st.clone())
    identical_step = all(torch.equal(a, b) for a, b in zip(outs["bounded_problem"], outs["weighted"]))
    times = {n: [] for n in bset}
    q = q0.clone()
    for _ in range(args.reps):
        for name, bd in bset.items():
            ev[0].record()
            for _ in range(args.steps):
                prob.step(q, ft0, pt, None, bounds=bd, **skw)
            ev[1].record()
            torch.cuda.synchronize()
            times[name].append(ev[0].elapsed_time(ev[1]) / args.steps)
    med = {n: float(np.median(v)) for n, v in times.items()}
    print(json.dumps({
        "part": "step", "workload": "g1", "B": B, "nv": nv, "steps_per_window": args.steps, "card": gpu,
        "identical_outputs": identical_step, "ms_per_step": {n: round(v, 4) for n, v in med.items()},
        "ms_per_step_all": {n: [round(x, 4) for x in v] for n, v in times.items()},
        "overhead_problem_bounds_pct": round(100 * (med["bounded_problem"] / med["weighted"] - 1), 2),
        "overhead_random_pct": round(100 * (med["bounded_random"] / med["weighted"] - 1), 2),
        "bounds_bytes_per_step": 3 * B * nv * 4,
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
    tkw = dict(dt=wl["dt"], damping=wl["damping"], weights=tw1, **CONV)

    def run_track(bd):
        q = q0.clone()
        ev[0].record()
        q_traj, it, st_, passes = prob.track(q, ft, ptt, None, bounds=bd, **tkw)
        ev[1].record()
        torch.cuda.synchronize()
        return ev[0].elapsed_time(ev[1]), q_traj, it, st_, int(passes)

    first = {n: run_track(bd) for n, bd in bset.items()}   # warm-up (graphs, workspace) and the outputs
    identical_track = all(torch.equal(a, b) for a, b in zip(first["bounded_problem"][1:4], first["weighted"][1:4]))
    ttimes = {n: [] for n in bset}
    passes = {n: first[n][4] for n in bset}
    for _ in range(args.reps):
        for name, bd in bset.items():
            ttimes[name].append(run_track(bd)[0])
    tmed = {n: float(np.median(v)) for n, v in ttimes.items()}
    print(json.dumps({
        "part": "track", "workload": "g1", "B": B, "T": T, "nv": nv, **CONV, "card": gpu, "identical_outputs": identical_track,
        "track_ms": {n: round(v, 2) for n, v in tmed.items()}, "track_ms_all": {n: [round(x, 2) for x in v] for n, v in ttimes.items()},
        "passes": passes, "ms_per_pass": {n: round(tmed[n] / passes[n], 4) for n in tmed},
        "overhead_problem_bounds_pct": round(100 * (tmed["bounded_problem"] / tmed["weighted"] - 1), 2),
    }), flush=True)


if __name__ == "__main__":
    main()
