#!/usr/bin/env python3
"""Cost of the per-body contact forces (rsb_batch_set_contact_bodies) on bench.py's config 3 (4096 ANYmal-like environments on the
513 x 513 height map, 4 sub-steps per control step, targets resident in HBM) and config 2 (fallen robots under random torques).

Median ms per control step, CUDA events on the batch's stream, L2 evicted before every timed iteration as bench.py does.  Modes,
each a batch of its own on the same seeded workload, settled before anything is timed:
  parent        another build of the library (--parent-lib: the commit before the feature), no contact bodies
  none          this library, no contact bodies: the step must cost what it did
  feet          the 4 feet listed
  all           all 13 bodies listed
  all+read      all 13 listed and rsb_batch_get_body_contact_forces into torch CUDA tensors after every step (two copies, no launch)
Each mode is warmed up and timed three times, alternating with the others in one process; the spread of `none` over its three runs is
the yardstick for every difference.  The card's name, power limit and SM clock are read in the same run.
usage: python tools/contact_force_probe.py [--parent-lib PATH] [--steps K] [--warmup W] [--out FILE.json]"""
import argparse
import importlib.util
import json
import os
import subprocess
import sys

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

import torch  # noqa: E402
import raisimlib_b200  # noqa: E402
from raisimlib_b200 import capi  # noqa: E402
from bench import GpuSim, Workload, L2_FLUSH_BYTES  # noqa: E402

FEET = ["LF_FOOT", "RF_FOOT", "LH_FOOT", "RH_FOOT"]


def load_capi(lib_path):
    """a second instance of the ctypes binding on another build of the library"""
    os.environ["RSB_LIB_PATH"] = lib_path
    try:
        spec = importlib.util.spec_from_file_location("raisimlib_b200_capi_parent", os.path.join(ROOT, "raisimlib_b200", "capi.py"))
        mod = importlib.util.module_from_spec(spec)
        spec.loader.exec_module(mod)
        mod.lib()
    finally:
        del os.environ["RSB_LIB_PATH"]
    return mod


def make_sim(wl, stream, binding):
    raisimlib_b200.capi = binding           # GpuSim takes the binding from the package
    try:
        return GpuSim(wl, 0, stream)
    finally:
        raisimlib_b200.capi = capi


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--parent-lib")
    ap.add_argument("--steps", type=int, default=200)
    ap.add_argument("--warmup", type=int, default=20)
    ap.add_argument("--envs", type=int, default=4096)
    ap.add_argument("--out")
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("contact_force_probe.py needs a CUDA device")
    capi.lib()
    parent = load_capi(os.path.abspath(args.parent_lib)) if args.parent_lib else None
    stream = torch.cuda.current_stream()
    n = args.envs
    flush = torch.empty(L2_FLUSH_BYTES // 4, dtype=torch.float32, device="cuda")
    force, steps_t = torch.empty((n, 13, 3), device="cuda"), torch.empty((n, 13), dtype=torch.int32, device="cuda")
    modes = (["parent"] if parent else []) + ["none", "feet", "all", "all+read"]
    res = {"device": torch.cuda.get_device_name(0), "steps": args.steps, "configs": {}}
    for key in ("c3", "c2"):
        wl = Workload(key, 0, n)
        sims = {}
        for m in modes:
            sim = sims[m] = make_sim(wl, stream, parent if m == "parent" else capi)
            if m == "feet":
                sim.bt.set_contact_bodies_by_name(FEET)
            elif m.startswith("all"):
                sim.bt.set_contact_bodies(list(range(13)))
            for k in range(wl.settle):
                sim.step_resident(k)
        counter = {m: wl.settle for m in modes}

        def run(m):
            sims[m].step_resident(counter[m]); counter[m] += 1
            if m == "all+read":
                sims[m].bt.body_contact_forces_into(force, steps_t)

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
        for _ in range(3):
            for m in modes:
                runs[m].append(timed(m))
        # the same seeded workload in every batch: listing bodies must not have changed a single state bit
        g0 = sims["none"].bt.get_state()[0]
        same = {m: bool(sims[m].bt.get_state()[0].tobytes() == g0.tobytes()) for m in modes}
        f, s = sims["all"].bt.body_contact_forces()
        med = {m: float(np.median(v)) for m, v in runs.items()}
        res["configs"][key] = {"workload": wl.name, "median_ms": med, "runs_ms": runs, "state_equal_to_none": same,
                               "spread_none": (max(runs["none"]) - min(runs["none"])) / med["none"],
                               "mean_bodies_in_contact": float((s > 0).sum(1).mean()), "mean_total_force_z": float(f[:, :, 2].sum(1).mean())}
        print(f"--- {key}: {wl.name}")
        for m in modes:
            print(f"{m:9s} {med[m]:.4f} ms  ({100 * (med[m] / med['none'] - 1):+.2f} % vs none; runs {', '.join(f'{x:.4f}' for x in runs[m])}; state equal {same[m]})")
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
