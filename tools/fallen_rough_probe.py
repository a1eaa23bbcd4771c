"""Cost of stage B's full-reach height-map search where it runs: ANYmal-like robots lying fallen on a rough 0.05 m map, so that
trunks, hips and shanks (radii and half extents of one to six pitches) sit on the terrain at every sub-step.

    python tools/fallen_rough_probe.py [--envs 4096] [--steps 200]

Prints one JSON line: ms per control step (4 sub-steps, host clock around device-synchronised launches, after warm-up), mean contacts per environment, the card and
its power limit.  RSB_LIB_PATH=other/librsb.so times another build of the library (an A/B comparison, one process each).
"""
import argparse
import json
import os
import subprocess
import sys
import time

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--envs", type=int, default=4096)
    ap.add_argument("--steps", type=int, default=200)
    ap.add_argument("--warmup", type=int, default=20)
    a = ap.parse_args()
    import torch
    from raisimlib_b200 import capi, RSC_DIR
    rng = np.random.default_rng(0)
    xs = ys = 513
    size = 25.6                                                        # pitch 0.05 m
    H = (0.06 * rng.uniform(-1, 1, (ys, xs))).astype(np.float32)
    m = capi.Model(os.path.join(RSC_DIR, "anymal_c_like.urdf"))
    n = a.envs
    bt = capi.Batch(m, n)
    bt.set_heightmap(xs, ys, size, size, 0.0, 0.0, H)
    gc = np.zeros((n, 19), np.float32)
    gc[:, 0:2] = rng.uniform(-0.4 * size, 0.4 * size, (n, 2))
    gc[:, 2] = 0.25
    q = rng.standard_normal((n, 4)); gc[:, 3:7] = q / np.linalg.norm(q, axis=1, keepdims=True)   # any orientation: fallen
    gc[:, 7:] = rng.uniform(-0.5, 0.5, (n, 12))
    bt.set_pd_gains(np.r_[np.zeros(6), 80.0 * np.ones(12)], np.r_[np.zeros(6), 2.0 * np.ones(12)])
    bt.set_pd_target(gc, np.zeros((n, 18), np.float32))
    bt.set_state(gc, np.zeros((n, 18), np.float32))
    for _ in range(a.warmup):
        bt.integrate(4)
    torch.cuda.synchronize()                                           # the whole device: the batch runs on a stream of its own
    t0 = time.perf_counter()
    for _ in range(a.steps):
        bt.integrate(4)
    torch.cuda.synchronize()
    ms = 1e3 * (time.perf_counter() - t0) / a.steps
    _, cnt = bt.contacts()
    card = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True, text=True).stdout.strip()
    print(json.dumps(dict(ms_per_control_step=round(ms, 4), envs=n, contacts_per_env=round(float(cnt.mean()), 2), gpu=card)))


if __name__ == "__main__":
    main()
