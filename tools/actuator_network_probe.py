#!/usr/bin/env python3
"""Cost of the learned actuator network (rsb_batch_set_actuator_network) on bench.py's config 3 (4096 ANYmal-like environments on the
513 x 513 height map, 4 sub-steps per control step).

Median ms per control step, CUDA events on the batch's stream, L2 evicted before every timed iteration as bench.py does.  Modes, each a
batch of its own on the same seeded workload, settled before anything is timed:
  parent   another build of the library (--parent-lib: the commit before the feature), PD law: the step without a network must cost
           what it did
  pd       this library, PD law on the 12 joints (no network)
  limp     this library, per-environment actuator rows kp = kd = 0 on the 12 joints: no joint torque, the robots sag
  net      this library, a network on the 12 joints (history 3, 3 hidden layers of 32, dense random hidden weights) whose output layer
           is zero: every weight is loaded and multiplied at every sub-step, and the torque is exactly that of `limp`, so the states
           of `net` and `limp` agree bit for bit and their difference is the cost of evaluating the network
Each mode is warmed up and timed --repeats times, alternating with the others in one process; the spread of every mode over its runs
is the yardstick for every difference.  The card's name, power limit and SM clock are read in the same run.
usage: python tools/actuator_network_probe.py [--parent-lib PATH] [--steps K] [--warmup W] [--repeats R] [--out FILE.json]"""
import argparse
import json
import os
import subprocess
import sys

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tools"))

import torch  # noqa: E402
from bench import Workload, L2_FLUSH_BYTES  # noqa: E402
from contact_force_probe import load_capi, make_sim  # noqa: E402
from raisimlib_b200 import capi  # noqa: E402

HISTORY, LAYERS, WIDTH = 3, 3, 32


def zero_output_network(rng):
    """[(W, b)]: dense random hidden layers, zero output layer (net = 0 exactly)"""
    out, nin = [], 2 * HISTORY
    for _ in range(LAYERS):
        out.append((rng.uniform(-1, 1, (WIDTH, nin)) / np.sqrt(nin), rng.uniform(-0.3, 0.3, WIDTH)))
        nin = WIDTH
    out.append((np.zeros((1, WIDTH)), np.zeros(1)))
    return [(w.astype(np.float32), b.astype(np.float32)) for w, b in out]


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--parent-lib")
    ap.add_argument("--steps", type=int, default=200)
    ap.add_argument("--warmup", type=int, default=20)
    ap.add_argument("--repeats", type=int, default=5)
    ap.add_argument("--envs", type=int, default=4096)
    ap.add_argument("--out")
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("actuator_network_probe.py needs a CUDA device")
    capi.lib()
    parent = load_capi(os.path.abspath(args.parent_lib)) if args.parent_lib else None
    stream = torch.cuda.current_stream()
    n = args.envs
    flush = torch.empty(L2_FLUSH_BYTES // 4, dtype=torch.float32, device="cuda")
    modes = (["parent"] if parent else []) + ["pd", "limp", "net"]
    res = {"device": torch.cuda.get_device_name(0), "steps": args.steps, "repeats": args.repeats,
           "network": dict(dofs=12, history=HISTORY, layers=LAYERS, width=WIDTH)}
    wl = Workload("c3", 0, n)
    layers = zero_output_network(np.random.default_rng(0))
    sims = {}
    for m in modes:
        sim = sims[m] = make_sim(wl, stream, parent if m == "parent" else capi)
        if m == "limp":
            rows = np.full((n, 18, 3), -1.0, np.float32); rows[:, 6:, :2] = 0.0
            sim.bt.set_actuator_params(rows)
        if m == "net":
            sim.bt.set_actuator_network(list(range(6, 18)), layers, HISTORY)
        for k in range(wl.settle):
            sim.step_resident(k)
    counter = {m: wl.settle for m in modes}

    def run(m):
        sims[m].step_resident(counter[m]); counter[m] += 1

    def timed(m):
        for _ in range(args.warmup):
            run(m)
        ev = [(torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)) for _ in range(args.steps)]
        torch.cuda.synchronize()
        for k in range(args.steps):
            flush.fill_(float(k))
            ev[k][0].record(stream)
            run(m)
            ev[k][1].record(stream)
        torch.cuda.synchronize()
        return float(np.median([a.elapsed_time(b) for a, b in ev]))

    runs = {m: [] for m in modes}
    for _ in range(args.repeats):
        for m in modes:
            runs[m].append(timed(m))
    g0, g1 = sims["pd"].bt.get_state()[0], sims["limp"].bt.get_state()[0]
    same = {m: bool(sims[m].bt.get_state()[0].tobytes() == g0.tobytes()) for m in modes}
    res["net_state_equal_to_limp"] = bool(sims["net"].bt.get_state()[0].tobytes() == g1.tobytes())
    med = {m: float(np.median(v)) for m, v in runs.items()}
    spread = {m: (max(v) - min(v)) / med[m] for m, v in runs.items()}
    res.update(workload=wl.name, median_ms=med, runs_ms=runs, spread=spread, state_equal_to_pd=same)
    print(f"--- c3: {wl.name}")
    for m in modes:
        print(f"{m:7s} {med[m]:.4f} ms  ({100 * (med[m] / med['pd'] - 1):+.2f} % vs pd; runs {', '.join(f'{x:.4f}' for x in runs[m])}; "
              f"spread {100 * spread[m]:.2f} %; state equal to pd {same[m]})")
    res["nvidia_smi"] = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm,clocks.sm", "--format=csv,noheader", "-i", "0"],
                                       capture_output=True, text=True).stdout.strip()
    print(f"net against limp: {1e3 * (med['net'] - med['limp']):+.1f} us per control step, states equal {res['net_state_equal_to_limp']}")
    print(res["nvidia_smi"])
    print(json.dumps(res))
    if args.out:
        with open(args.out, "w") as f:
            json.dump(res, f, indent=1)


if __name__ == "__main__":
    main()
