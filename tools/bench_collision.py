"""What per-instance collision avoidance costs, and what a sparse pair mask saves (needs a GPU).

  python tools/bench_collision.py [--steps 100] [--reps 5]

Two collision workloads at the sizes the README quotes: "aloha_coll" (1 104 geom pairs) at 1 024 instances and "ur5e_wall"
(the wrist against a floor and a wall) at 16 384, fp32 inputs (K1 runs in fp64 for collision problems), in one process.
Three variants, alternating window by window:

  bounded  the entry points without collision arguments (bik_step / bik_converge: what bik_step_coll with a null `coll` runs)
  ones     bik_step_coll / bik_converge_coll with an all-ones pair mask (the same QPs: what reading the mask costs)
  sparse   the same with 10 % of the pairs enabled per instance (seeded; at least one): the distances of the others are
           never computed, and the QPs have fewer rows

step      one call per step, `steps` calls per timed window (CUDA events); then the same windows with BIK_STEP_PHASE=1, which
          runs K1 alone, to separate what the mask changes in K1.
converge  bik_converge / bik_converge_coll from the same q0 (max_iters 20, thresholds 1e-3), one call per window.

The all-ones variant must give the outputs of the variant without collision arguments bit for bit; the script checks that.
Prints one JSON line per workload and part: median times, every repetition, the overhead of the all-ones mask, what the
sparse mask saves, the card and its power limit.
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

CONV = dict(max_iters=20, pos_threshold=1e-3, ori_threshold=1e-3)
CASES = [("aloha_coll", 1024), ("ur5e_wall", 16384)]


def card():
    try:
        out = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader", "-i", "0"],
                             capture_output=True, text=True, timeout=30).stdout.strip()
    except (OSError, subprocess.TimeoutExpired):
        out = ""
    return out or torch.cuda.get_device_name(0)


def bench(name, B, args, gpu, ev):
    wl = WORKLOADS[name]
    fm = load_flat(wl["robot"])
    spec = spec_from_workload(fm, wl)
    model = DeviceModel(fm, 0)
    prob = Problem(model, spec)
    frames = task_frames(wl, fm)
    dev, npairs, nv = "cuda:0", prob.npairs, fm.nv

    def fk(qq):
        p, c = model.fk(qq, frames, want_com=bool(spec.ncom))
        return p.cpu().numpy().astype(np.float64), (None if c is None else c.cpu().numpy().astype(np.float64))

    inp = make_inputs(fm, wl, B, fk, seed=1000)
    q0 = torch.tensor(inp["q"], dtype=torch.float32, device=dev)
    ft = torch.tensor(inp["frame_targets"], dtype=torch.float32, device=dev)
    pt = None if inp.get("posture_target") is None else torch.tensor(inp["posture_target"], dtype=torch.float32, device=dev)
    ct = None if inp.get("com_target") is None else torch.tensor(inp["com_target"], dtype=torch.float32, device=dev)
    rng = np.random.default_rng(11)
    sparse = rng.uniform(size=(B, npairs)) < 0.1
    sparse[np.arange(B), rng.integers(0, npairs, size=B)] = True
    variants = {"bounded": None, "ones": (torch.ones((B, npairs), dtype=torch.uint8, device=dev), None, None),
                "sparse": (torch.tensor(sparse.astype(np.uint8), device=dev), None, None)}
    dq = torch.empty((B, nv), device=dev)
    st = torch.empty(B, device=dev, dtype=torch.int32)
    skw = dict(dt=wl["dt"], damping=wl["damping"], dq=dq, status=st)
    outs = {}
    for v, co in variants.items():   # warm-up, and the outputs of one step from q0
        prob.step(q0.clone(), ft, pt, ct, collision=co, **skw)
        torch.cuda.synchronize()
        outs[v] = (dq.clone(), st.clone())
    identical_step = all(torch.equal(a, b) for a, b in zip(outs["ones"], outs["bounded"]))

    def windows(phase):
        if phase:
            os.environ["BIK_STEP_PHASE"] = phase
        try:
            times = {v: [] for v in variants}
            q = q0.clone()
            for _ in range(args.reps):
                for v, co in variants.items():
                    ev[0].record()
                    for _ in range(args.steps):
                        prob.step(q, ft, pt, ct, collision=co, **skw)
                    ev[1].record()
                    torch.cuda.synchronize()
                    times[v].append(ev[0].elapsed_time(ev[1]) / args.steps)
            return times
        finally:
            os.environ.pop("BIK_STEP_PHASE", None)

    step_t, k1_t = windows(None), windows("1")
    med = lambda t: {v: float(np.median(x)) for v, x in t.items()}
    sm, km = med(step_t), med(k1_t)
    print(json.dumps({
        "part": "step", "workload": name, "B": B, "npairs": npairs, "enabled_sparse": round(float(sparse.mean()), 4),
        "steps_per_window": args.steps, "card": gpu, "identical_outputs": identical_step,
        "ms_per_step": {v: round(x, 4) for v, x in sm.items()}, "ms_per_step_all": {v: [round(x, 4) for x in t] for v, t in step_t.items()},
        "k1_ms_per_step": {v: round(x, 4) for v, x in km.items()}, "k1_ms_all": {v: [round(x, 4) for x in t] for v, t in k1_t.items()},
        "overhead_ones_pct": round(100 * (sm["ones"] / sm["bounded"] - 1), 2),
        "k1_overhead_ones_pct": round(100 * (km["ones"] / km["bounded"] - 1), 2),
        "sparse_saves_step_pct": round(100 * (1 - sm["sparse"] / sm["bounded"]), 2),
        "sparse_saves_k1_pct": round(100 * (1 - km["sparse"] / km["bounded"]), 2),
    }), flush=True)

    def run_conv(co):
        q = q0.clone()
        ev[0].record()
        it, st_ = prob.converge(q, ft, pt, ct, collision=co, dt=wl["dt"], damping=wl["damping"], **CONV)
        ev[1].record()
        torch.cuda.synchronize()
        return ev[0].elapsed_time(ev[1]), q, it, st_

    first = {v: run_conv(co) for v, co in variants.items()}   # warm-up (graphs, workspace) and the outputs
    identical_conv = all(torch.equal(a, b) for a, b in zip(first["ones"][1:], first["bounded"][1:]))
    ctimes = {v: [] for v in variants}
    for _ in range(args.reps):
        for v, co in variants.items():
            ctimes[v].append(run_conv(co)[0])
    cm = med(ctimes)
    print(json.dumps({
        "part": "converge", "workload": name, "B": B, "npairs": npairs, **CONV, "card": gpu, "identical_outputs": identical_conv,
        "converge_ms": {v: round(x, 3) for v, x in cm.items()}, "converge_ms_all": {v: [round(x, 3) for x in t] for v, t in ctimes.items()},
        "mean_iters": {v: round(float(first[v][2].float().mean()), 2) for v in variants},
        "overhead_ones_pct": round(100 * (cm["ones"] / cm["bounded"] - 1), 2),
        "sparse_saves_pct": round(100 * (1 - cm["sparse"] / cm["bounded"]), 2),
    }), flush=True)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--steps", type=int, default=100)
    ap.add_argument("--reps", type=int, default=5)
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("bench_collision.py needs a CUDA device")
    gpu = card()
    ev = [torch.cuda.Event(enable_timing=True) for _ in range(2)]
    for name, B in CASES:
        bench(name, B, args, gpu, ev)


if __name__ == "__main__":
    main()
