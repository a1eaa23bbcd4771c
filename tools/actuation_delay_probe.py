#!/usr/bin/env python3
"""Cost of the actuation delay (rsb_batch_set_actuation_delay) on bench.py's config 3 (4096 ANYmal-like environments on the 513 x 513
height map) and config 4 (4096 Atlas-like humanoids on flat ground), 4 sub-steps per control step.

Median ms per control step, CUDA events on the batch's stream, L2 evicted before every timed iteration as bench.py does.  Modes, each a
batch of its own on the same seeded workload, settled before anything is timed:
  parent   another build of the library (--parent-lib: the commit before the feature): the step without a delay must cost what it did
  none     this library, no delay set
  zeros    this library, every delay 0: the delay instance of the step runs, and the state equals that of `none` bit for bit
  u0_8     this library, delays drawn from U{0..8} sub-steps per environment
Each mode is warmed up and timed --repeats times, alternating with the others in one process; the spread of every mode over its runs
is the yardstick for every difference.  The card's name, power limit and SM clock are read in the same run.
usage: python tools/actuation_delay_probe.py [--parent-lib PATH] [--steps K] [--warmup W] [--repeats R] [--out FILE.json]"""
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


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--parent-lib")
    ap.add_argument("--steps", type=int, default=200)
    ap.add_argument("--warmup", type=int, default=20)
    ap.add_argument("--repeats", type=int, default=4)
    ap.add_argument("--envs", type=int, default=4096)
    ap.add_argument("--configs", default="c3,c4")
    ap.add_argument("--out")
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("actuation_delay_probe.py needs a CUDA device")
    capi.lib()
    parent = load_capi(os.path.abspath(args.parent_lib)) if args.parent_lib else None
    stream = torch.cuda.current_stream()
    n = args.envs
    flush = torch.empty(L2_FLUSH_BYTES // 4, dtype=torch.float32, device="cuda")
    modes = (["parent"] if parent else []) + ["none", "zeros", "u0_8"]
    res = {"device": torch.cuda.get_device_name(0), "steps": args.steps, "repeats": args.repeats, "configs": {}}
    for key in args.configs.split(","):
        wl = Workload(key, 0, n)
        sims = {}
        for m in modes:
            sim = sims[m] = make_sim(wl, stream, parent if m == "parent" else capi)
            if m == "zeros":
                sim.bt.set_actuation_delay(np.zeros(n, np.int32))
            if m == "u0_8":
                sim.bt.set_actuation_delay(np.random.default_rng(0).integers(0, 9, n).astype(np.int32))
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
        g0 = sims["none"].bt.get_state()[0]
        same = {m: bool(sims[m].bt.get_state()[0].tobytes() == g0.tobytes()) for m in modes}
        med = {m: float(np.median(v)) for m, v in runs.items()}
        spread = {m: (max(v) - min(v)) / med[m] for m, v in runs.items()}
        res["configs"][key] = dict(workload=wl.name, median_ms=med, runs_ms=runs, spread=spread, state_equal_to_none=same)
        print(f"--- {key}: {wl.name}")
        for m in modes:
            print(f"{m:7s} {med[m]:.4f} ms  ({100 * (med[m] / med['none'] - 1):+.2f} % vs none; runs {', '.join(f'{x:.4f}' for x in runs[m])}; "
                  f"spread {100 * spread[m]:.2f} %; state equal to none {same[m]})")
        del sims
    res["nvidia_smi"] = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm,clocks.sm", "--format=csv,noheader", "-i", "0"],
                                       capture_output=True, text=True).stdout.strip()
    print(res["nvidia_smi"])
    print(json.dumps(res))
    if args.out:
        with open(args.out, "w") as f:
            json.dump(res, f, indent=1)


if __name__ == "__main__":
    main()
