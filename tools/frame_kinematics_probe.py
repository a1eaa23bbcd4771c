#!/usr/bin/env python3
"""Cost of the frame getters on the headline workload of bench.py (BASELINE config 3: 4096 ANYmal-like environments on the 513 x 513
height map, 4 sub-steps per control step, targets resident in HBM), frames = base + 4 feet, outputs into torch CUDA tensors.

Median ms per control step, CUDA events on the batch's stream, L2 evicted before every timed iteration as bench.py does:
  step                 the control step alone
  step+states          + rsb_batch_get_frame_states (kinematics pass + frame kernel: the poses are stale after a step)
  step+states+jac      + rsb_batch_get_frame_jacobians (frame kernel only: the poses are current)
  kinematics           rsb_batch_update_kinematics alone
  states_kernel        the frame kernel writing the states (poses current)
  jac_kernel           the frame kernel writing the Jacobians (poses current)
Each mode is warmed up and timed three times, alternating with the others; the card's name and power limit are read in the same run.
usage: python tools/frame_kinematics_probe.py [--steps K] [--warmup W] [--out FILE.json]"""
import argparse
import json
import os
import subprocess
import sys

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

import torch  # noqa: E402
from bench import GpuSim, Workload, L2_FLUSH_BYTES  # noqa: E402

FRAMES = ["base", "LF_FOOT", "RF_FOOT", "LH_FOOT", "RH_FOOT"]
MODES = ["step", "step+states", "step+states+jac", "kinematics", "states_kernel", "jac_kernel"]


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--steps", type=int, default=200)
    ap.add_argument("--warmup", type=int, default=20)
    ap.add_argument("--envs", type=int, default=4096)
    ap.add_argument("--out")
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("frame_kinematics_probe.py needs a CUDA device")
    stream = torch.cuda.current_stream()
    wl = Workload("c3", 0, args.envs)
    sim = GpuSim(wl, 0, stream)
    bt, n = sim.bt, args.envs
    bt.set_frames_by_name(FRAMES)
    F = len(FRAMES)
    pos, lin, ang = (torch.empty((n, F, 3), device="cuda") for _ in range(3))
    rot = torch.empty((n, F, 3, 3), device="cuda")
    jac = torch.empty((n, F, 6, bt.nv), device="cuda")
    flush = torch.empty(L2_FLUSH_BYTES // 4, dtype=torch.float32, device="cuda")
    for k in range(wl.settle):                 # robots dropped onto the terrain stand before anything is timed (as in bench.py)
        sim.step_resident(k)
    step = [wl.settle]

    def run(mode):
        if mode.startswith("step"):
            sim.step_resident(step[0]); step[0] += 1
            if "states" in mode:
                bt.frame_states_into(pos, rot, lin, ang)
            if "jac" in mode:
                bt.frame_jacobians_into(jac)
        elif mode == "kinematics":
            bt.update_kinematics()
        elif mode == "states_kernel":
            bt.frame_states_into(pos, rot, lin, ang)
        else:
            bt.frame_jacobians_into(jac)

    def timed(mode):
        if not mode.startswith("step"):
            bt.update_kinematics()             # the kernel-only modes run on current poses
        for _ in range(args.warmup):
            run(mode)
        l0 = bt.launch_count()
        ev = [(torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)) for _ in range(args.steps)]
        torch.cuda.synchronize()
        for k in range(args.steps):
            flush.fill_(float(k))
            ev[k][0].record(stream)
            run(mode)
            ev[k][1].record(stream)
        torch.cuda.synchronize()
        return float(np.median([a.elapsed_time(b) for a, b in ev])), (bt.launch_count() - l0) / args.steps

    runs = {m: [] for m in MODES}
    launches = {}
    for _ in range(3):
        for m in MODES:
            ms, launches[m] = timed(m)
            runs[m].append(ms)
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader", "-i", "0"],
                       capture_output=True, text=True).stdout.strip()
    res = {"device": torch.cuda.get_device_name(0), "nvidia_smi": q, "workload": wl.name, "frames": FRAMES, "steps": args.steps,
           "median_ms": {m: float(np.median(v)) for m, v in runs.items()}, "runs_ms": runs, "launches_per_iteration": launches}
    for m in MODES:
        print(f"{m:18s} {res['median_ms'][m]:.4f} ms  (runs {', '.join(f'{x:.4f}' for x in runs[m])}; launches {launches[m]:.0f})")
    print(json.dumps(res))
    if args.out:
        with open(args.out, "w") as f:
            json.dump(res, f, indent=1)


if __name__ == "__main__":
    main()
