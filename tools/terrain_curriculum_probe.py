#!/usr/bin/env python3
"""Cost of the terrain curriculum calls at 4096 ANYmal-like environments on a 16-map atlas of bench.py's 513 x 513 height map size,
host wall time per call (each call waits for its device check, so that is what the caller pays), after warm-up, nothing else queued:
  index_host     rsb_batch_set_heightmap_index of all environments from a pageable numpy array
  index_device   the same from a torch CUDA int32 tensor
  update_host    rsb_batch_update_heightmaps of one 513 x 513 map from a pageable numpy array
  update_device  the same from a torch CUDA float32 tensor
  atlas_16       for comparison, the route without these calls: rsb_batch_set_heightmaps of the whole 16-map atlas and index
Each mode is timed --repeats times, alternating in one process; medians and the spread over the runs are printed.  The card's name,
power limit and SM clock are read in the same run.
usage: python tools/terrain_curriculum_probe.py [--calls K] [--warmup W] [--repeats R] [--envs N] [--out FILE.json]"""
import argparse
import json
import os
import subprocess
import sys
import time

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

import torch  # noqa: E402
from bench import HM  # noqa: E402
from raisimlib_b200 import capi, RSC_DIR  # noqa: E402


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--calls", type=int, default=100)
    ap.add_argument("--warmup", type=int, default=10)
    ap.add_argument("--repeats", type=int, default=5)
    ap.add_argument("--envs", type=int, default=4096)
    ap.add_argument("--maps", type=int, default=16)
    ap.add_argument("--out")
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("terrain_curriculum_probe.py needs a CUDA device")
    n, L = args.envs, args.maps
    rng = np.random.default_rng(3)
    H = rng.uniform(-0.1, 0.1, (L, HM["ys"], HM["xs"])).astype(np.float32)
    idx = [rng.integers(0, L, n).astype(np.int32) for _ in range(4)]
    didx = [torch.from_numpy(x).cuda() for x in idx]
    one, done = H[3:4].copy(), torch.from_numpy(H[3:4]).cuda()
    m = capi.Model(os.path.join(RSC_DIR, "anymal_c_like.urdf"))
    bt = capi.Batch(m, n)
    bt.set_stream(torch.cuda.current_stream().cuda_stream)
    bt.set_heightmaps(HM["size"], HM["size"], 0.0, 0.0, H, idx[0])
    counter = [0]

    def run(mode):
        k = counter[0] = counter[0] + 1
        if mode == "index_host":
            bt.set_heightmap_index(idx[k % 4])
        elif mode == "index_device":
            bt.set_heightmap_index_from(didx[k % 4])
        elif mode == "update_host":
            bt.update_heightmaps(3, one)
        elif mode == "update_device":
            bt.update_heightmaps_from(3, done)
        else:
            bt.set_heightmaps(HM["size"], HM["size"], 0.0, 0.0, H, idx[k % 4])

    def timed(mode):
        for _ in range(args.warmup):
            run(mode)
        torch.cuda.synchronize()
        l0 = bt.launch_count()
        t = []
        for _ in range(args.calls):
            t0 = time.perf_counter(); run(mode); t.append(time.perf_counter() - t0)
        torch.cuda.synchronize()
        assert bt.launch_count() == l0
        return 1e3 * float(np.median(t))

    modes = ["index_host", "index_device", "update_host", "update_device", "atlas_16"]
    runs = {md: [] for md in modes}
    for _ in range(args.repeats):
        for md in modes:
            runs[md].append(timed(md))
    med = {md: float(np.median(v)) for md, v in runs.items()}
    spread = {md: (max(v) - min(v)) / med[md] for md, v in runs.items()}
    res = {"device": torch.cuda.get_device_name(0), "envs": n, "maps": L, "map": [HM["ys"], HM["xs"]], "calls": args.calls,
           "repeats": args.repeats, "median_ms": med, "runs_ms": runs, "spread": spread}
    print(f"--- {n} environments, atlas of {L} maps of {HM['xs']} x {HM['ys']}: host wall time per call")
    for md in modes:
        print(f"{md:14s} {med[md]:.4f} ms  (runs {', '.join(f'{x:.4f}' for x in runs[md])}; spread {100 * spread[md]:.2f} %)")
    res["nvidia_smi"] = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm,clocks.sm", "--format=csv,noheader", "-i", "0"],
                                       capture_output=True, text=True).stdout.strip()
    print(res["nvidia_smi"])
    print(json.dumps(res))
    if args.out:
        with open(args.out, "w") as f:
            json.dump(res, f, indent=1)


if __name__ == "__main__":
    main()
