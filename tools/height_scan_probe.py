#!/usr/bin/env python3
"""Cost of the terrain height scan (rsb_batch_get_height_scan) at 4096 ANYmal-like environments on bench.py's 513 x 513 rough height
map, under the RaisimGym task (rsb_batch_gym_step, 4 sub-steps per control step), device-resident buffers, CUDA events on the batch's
stream after warm-up:
  scan_base   the scan kernel alone, 187 yaw-aligned base points (legged_gym's 11 x 17 grid): poses from gc, no kinematics pass
  scan_feet   the scan kernel alone, 52 points around each of the 4 feet (208): the kinematics pass ran once before timing, the state
              does not change in between, so each timed call is the scan launch only
  gym         ms per control step of gym_step
  gym_scan    ms per control step of gym_step followed by height_scan_into of the base grid (two launches)
Each mode is timed --repeats times, alternating in one process; medians and the spread over the runs are printed.  The card's name,
power limit and SM clock are read in the same run.
usage: python tools/height_scan_probe.py [--steps K] [--warmup W] [--repeats R] [--envs N] [--out FILE.json]"""
import argparse
import json
import os
import subprocess
import sys

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

import torch  # noqa: E402
from bench import HM, Workload  # noqa: E402
from raisimlib_b200 import capi, RSC_DIR  # noqa: E402


def base_grid():
    gx, gy = np.meshgrid(np.linspace(-0.8, 0.8, 11), np.linspace(-0.5, 0.5, 17), indexing="ij")
    return np.stack([gx.reshape(-1), gy.reshape(-1)], 1).astype(np.float32)


def foot_rings():
    """52 points per foot: rings of 8, 12, 16 and 16 points at radii 0.05 / 0.1 / 0.15 / 0.2 m"""
    pts = []
    for r, k in ((0.05, 8), (0.10, 12), (0.15, 16), (0.20, 16)):
        a = 2 * np.pi * np.arange(k) / k
        pts.append(np.stack([r * np.cos(a), r * np.sin(a)], 1))
    return np.concatenate(pts).astype(np.float32)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--steps", type=int, default=500)
    ap.add_argument("--warmup", type=int, default=50)
    ap.add_argument("--repeats", type=int, default=5)
    ap.add_argument("--envs", type=int, default=4096)
    ap.add_argument("--out")
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("height_scan_probe.py needs a CUDA device")
    n, substeps = args.envs, 4
    wl = Workload("c3", 0, n)
    gc0 = np.array([0, 0, 0.57, 1, 0, 0, 0, 0.03, 0.4, -0.8, -0.03, 0.4, -0.8, 0.03, -0.4, 0.8, -0.03, -0.4, 0.8])
    m = capi.Model(os.path.join(RSC_DIR, "anymal_c_like.urdf"))
    stream = torch.cuda.current_stream()
    feet = [m.body_index(f"{leg}_FOOT") for leg in ("LF", "RF", "LH", "RH")]
    grid, ring = base_grid(), foot_rings()

    def make(points):
        bt = capi.Batch(m, n)
        bt.set_stream(stream.cuda_stream)
        bt.set_heightmap(HM["xs"], HM["ys"], HM["size"], HM["size"], 0.0, 0.0, wl.H)
        bt.set_params(threshold=1e-6)
        bt.set_pd_gains(np.r_[np.zeros(6), 100.0 * np.ones(12)], np.r_[np.zeros(6), 2.0 * np.ones(12)])
        g0 = gc0.copy(); g0[2] = 0.57 + float(np.max(wl.H))
        bt.gym_configure(g0, np.zeros(18), g0[7:], 0.6 * np.ones(12), feet)
        bt.gym_reset()
        bt.set_height_scan(*points)
        return bt

    base_pts = (np.zeros(len(grid), np.int32), grid)
    foot_pts = (np.repeat(np.array(feet, np.int32), len(ring)), np.tile(ring, (4, 1)))
    g = torch.Generator(device="cuda"); g.manual_seed(7)
    acts = [0.15 * torch.randn((n, 12), device="cuda", generator=g) for _ in range(8)]
    obs = torch.empty((n, 34), device="cuda"); rew = torch.empty(n, device="cuda"); done = torch.empty(n, dtype=torch.uint8, device="cuda")
    sims = {"base": make(base_pts), "feet": make(foot_pts), "gym": make(base_pts)}
    for bt in sims.values():
        for k in range(30):
            bt.gym_step(acts[k % 8], substeps, obs, rew, done)
    hb, hf = torch.empty((n, len(grid)), device="cuda"), torch.empty((n, 4 * len(ring)), device="cuda")
    sims["feet"].height_scan_into(hf)              # the kinematics pass for the feet runs here, outside the timed loop
    counter = [30]

    def run(mode):
        if mode == "scan_base":
            sims["base"].height_scan_into(hb)
        elif mode == "scan_feet":
            sims["feet"].height_scan_into(hf)
        else:
            bt = sims["gym"]
            bt.gym_step(acts[counter[0] % 8], substeps, obs, rew, done); counter[0] += 1
            if mode == "gym_scan":
                bt.height_scan_into(hb)

    def timed(mode):
        for _ in range(args.warmup):
            run(mode)
        ev = [(torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)) for _ in range(args.steps)]
        torch.cuda.synchronize()
        l0 = sum(bt.launch_count() for bt in sims.values())
        for k in range(args.steps):
            ev[k][0].record(stream); run(mode); ev[k][1].record(stream)
        torch.cuda.synchronize()
        launches = (sum(bt.launch_count() for bt in sims.values()) - l0) / args.steps
        return float(np.median([a.elapsed_time(b) for a, b in ev])), launches

    modes = ["scan_base", "scan_feet", "gym", "gym_scan"]
    runs, per = {md: [] for md in modes}, {}
    for _ in range(args.repeats):
        for md in modes:
            t, per[md] = timed(md)
            runs[md].append(t)
    med = {md: float(np.median(v)) for md, v in runs.items()}
    spread = {md: (max(v) - min(v)) / med[md] for md, v in runs.items()}
    res = {"device": torch.cuda.get_device_name(0), "envs": n, "steps": args.steps, "repeats": args.repeats, "base_points": len(grid),
           "foot_points": 4 * len(ring), "median_ms": med, "runs_ms": runs, "spread": spread, "launches_per_call": per}
    print(f"--- {n} ANYmal-like environments, {HM['xs']} x {HM['ys']} rough map, gym_step of {substeps} sub-steps")
    for md in modes:
        print(f"{md:9s} {med[md]:.4f} ms  (launches per call {per[md]:.2f}; runs {', '.join(f'{x:.4f}' for x in runs[md])}; spread {100 * spread[md]:.2f} %)")
    print(f"gym_scan - gym: {med['gym_scan'] - med['gym']:+.4f} ms per control step ({100 * (med['gym_scan'] / med['gym'] - 1):+.2f} %)")
    res["nvidia_smi"] = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm,clocks.sm", "--format=csv,noheader", "-i", "0"],
                                       capture_output=True, text=True).stdout.strip()
    print(res["nvidia_smi"])
    print(json.dumps(res))
    if args.out:
        with open(args.out, "w") as f:
            json.dump(res, f, indent=1)


if __name__ == "__main__":
    main()
