#!/usr/bin/env python3
"""What the IMU readings cost the batched step, on tools/feature_cost.py's harness: the same options (--parent-lib, --configs, --envs,
--steps, --warmup, --repeats, --out), the same timing, modes alternated in one process.

    python tools/imu_cost.py [--parent-lib PATH] [--configs c3,c4] ...

Modes: `none` (no sensors), `base` (one sensor at the base origin), `eight` (eight sensors: the base, the four feet and three frames
off the thighs and shanks, one rotated), `base+read` (`base`, read into torch CUDA tensors after every control step).  With
--parent-lib the first mode also runs on the parent build, as `parent`.  Every mode's final state is compared with that of `none`.
"""
import os
import sys

import numpy as np
import torch

sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
import feature_cost  # noqa: E402

EIGHT = ([0, 3, 6, 9, 12, 2, 5, 8], [[0, 0, 0], [0, 0, 0], [0, 0, 0], [0, 0, 0], [0, 0, 0], [0.1, 0, -0.05], [0.05, 0.02, -0.1], [0, 0, 0]])


def imu(bt, mode, wl):
    if mode.startswith("base"):
        bt.set_imus([0], np.zeros((1, 3), np.float32))
    elif mode == "eight":
        rot = np.tile(np.eye(3, dtype=np.float32), (8, 1, 1))
        rot[7] = [[0, -1, 0], [1, 0, 0], [0, 0, 1]]
        bt.set_imus(EIGHT[0], np.array(EIGHT[1], np.float32), rot)
    if mode == "base+read":
        lin, ang = torch.empty((wl.n, 1, 3), device="cuda"), torch.empty((wl.n, 1, 3), device="cuda")
        return lambda: bt.imu_readings_into(lin, ang)


feature_cost.FEATURES["imu"] = dict(configs="c3,c4", modes=["none", "base", "eight", "base+read"], setup=feature_cost.per_mode(imu), ref="none")

if __name__ == "__main__":
    sys.argv[1:1] = ["imu"]
    feature_cost.main()
