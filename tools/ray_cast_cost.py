#!/usr/bin/env python3
"""What ray casts cost, on tools/feature_cost.py's harness: the same options (--configs, --envs, --steps, --warmup, --repeats, --out), the
same timing, modes alternated in one process.

    python tools/ray_cast_cost.py [--configs c3] [--envs 4096] ...

RaisimGym batches (rsb_batch_gym_step, 4 sub-steps per control step) on the config's height map, 30 control steps in:
  gym          gym_step alone
  cam_terrain  a 64 x 48 pinhole camera (87 degrees wide) on the front of the base, pitched 30 degrees down, seeing the terrain only:
               the ray kernel alone, poses from gc
  cam_all      the same camera also seeing the robot: the ray kernel alone; the state does not change between calls, so after the first
               warm-up call's kinematics pass each call is the ray launch only
  gym_cam      gym_step, then cam_all: the kinematics pass and the ray launch
  lidar        16 x 360 rays on the base (elevations -15 .. +15 degrees, 1 degree in azimuth), terrain only
Outputs go to torch CUDA tensors.  The summary gives the rays of one call (environments x rays), from which rays per second follow.
"""
import itertools
import os
import sys

import numpy as np
import torch

sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
import feature_cost  # noqa: E402
from feature_cost import FEET, GC0, HM, RSC_DIR, SUBSTEPS  # noqa: E402

MAX_DISTANCE = 10.0


def camera(binding):
    d = binding.pinhole_rays(64, 48, 87.0)
    a = np.radians(30.0)
    Ry = np.array([[np.cos(a), 0, np.sin(a)], [0, 1, 0], [-np.sin(a), 0, np.cos(a)]])
    d = d @ Ry.T
    return np.zeros(len(d), np.int32), np.tile([0.35, 0.0, 0.05], (len(d), 1)).astype(np.float32), d.astype(np.float32)


def lidar():
    el, az = np.radians(np.linspace(-15, 15, 16)), np.radians(np.arange(360.0))
    E, A = np.meshgrid(el, az, indexing="ij")
    d = np.stack([np.cos(E) * np.cos(A), np.cos(E) * np.sin(A), np.sin(E)], -1).reshape(-1, 3)
    return np.zeros(len(d), np.int32), np.tile([0.0, 0.0, 0.2], (len(d), 1)).astype(np.float32), d.astype(np.float32)


def ray_cast(wl, binding, modes):
    n, stream = wl.n, torch.cuda.current_stream()
    m = binding.Model(os.path.join(RSC_DIR, "anymal_c_like.urdf"))
    feet = [m.body_index(f) for f in FEET]
    g = torch.Generator(device="cuda")
    g.manual_seed(7)
    acts = [0.15 * torch.randn((n, 12), device="cuda", generator=g) for _ in range(8)]
    obs, rew, done = torch.empty((n, 34), device="cuda"), torch.empty(n, device="cuda"), torch.empty(n, dtype=torch.uint8, device="cuda")
    cam, lid = camera(binding), lidar()
    rays = {"gym": None, "cam_terrain": (cam, "terrain"), "cam_all": (cam, "all"), "gym_cam": (cam, "all"), "lidar": (lid, "terrain")}

    def gym_batch(r):
        bt = binding.Batch(m, n)
        bt.set_stream(stream.cuda_stream)
        bt.set_heightmap(HM["xs"], HM["ys"], HM["size"], HM["size"], 0.0, 0.0, wl.H)
        bt.set_params(threshold=1e-6)
        bt.set_pd_gains(np.r_[np.zeros(6), 100.0 * np.ones(12)], np.r_[np.zeros(6), 2.0 * np.ones(12)])
        g0 = GC0.copy()
        g0[2] = 0.57 + float(np.max(wl.H))
        bt.gym_configure(g0, np.zeros(18), g0[7:], 0.6 * np.ones(12), feet)
        bt.gym_reset()
        if r is not None:
            bt.set_rays(*r[0], MAX_DISTANCE, r[1])
        for k in range(30):
            bt.gym_step(acts[k % 8], SUBSTEPS, obs, rew, done)
        return bt

    bts = {md: gym_batch(rays[md]) for md in modes}
    out = {md: (torch.empty((n, len(rays[md][0][0])), device="cuda"), torch.empty((n, len(rays[md][0][0])), dtype=torch.int32, device="cuda"))
           for md in modes if rays[md] is not None}
    k = {md: itertools.count(30) for md in modes}

    def step(md):
        bts[md].gym_step(acts[next(k[md]) % 8], SUBSTEPS, obs, rew, done)

    runs = {"gym": lambda: step("gym"), "cam_terrain": lambda: bts["cam_terrain"].ray_casts_into(*out["cam_terrain"]),
            "cam_all": lambda: bts["cam_all"].ray_casts_into(*out["cam_all"]), "lidar": lambda: bts["lidar"].ray_casts_into(*out["lidar"]),
            "gym_cam": lambda: (step("gym_cam"), bts["gym_cam"].ray_casts_into(*out["gym_cam"]))}
    return {md: (runs[md], bts[md]) for md in modes}


def summary(batches):
    return {"rays_per_call": {md: bt.n * bt.nrays for md, bt in batches.items() if md != "gym" and md != "parent"},
            "max_distance": MAX_DISTANCE}


feature_cost.FEATURES["ray_cast"] = dict(configs="c3", modes=["gym", "cam_terrain", "cam_all", "gym_cam", "lidar"], setup=ray_cast,
                                         summary=summary)

if __name__ == "__main__":
    sys.argv[1:1] = ["ray_cast"]
    feature_cost.main()
