#!/usr/bin/env python3
"""What does self-collision cost, and how often does it fire?  (exploratory, not a bench value; needs one GPU)

Runs bench.py's config 2 (ANYmal-like robots fallen on flat ground under random joint torques) and config 4 (Atlas-like humanoids
standing on box feet under PD) in three arms each:
  * off       -- no pairs, the instance pick_config chooses by default (quadruped / humanoid),
  * generic   -- no pairs, the generic instance forced (RSB_FORCE_GENERIC=1): what routing alone costs,
  * on        -- the pairs below enabled (which routes to the generic instance),
and prints, per arm, ms per control step (CUDA events around each launch of 4 fused sub-steps, after the bench's settling steps), the
share of environments holding a self contact after the last step, the mean number of self contacts and the mean Gauss-Seidel sweeps,
with the device name and power limit read in the same process.

Pairs (collision-body indices of the two shipped models):
  config 2: ANYmal-like leg to leg -- knee spheres, foot spheres and thigh capsules of the left / right and front / hind neighbours,
            the two diagonal foot pairs, and each front foot against the other front knee (16 pairs);
  config 4: Atlas-like -- thigh capsules, knee spheres against each other, against the other thigh and the other foot box; hands against
            the upper torso, the pelvis and each other; the head against both hands (13 pairs).
"""
import json
import os
import sys

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
import torch  # noqa: E402

import bench  # noqa: E402

ANYMAL = {"LF": (2, 3, 4), "RF": (6, 7, 8), "LH": (10, 11, 12), "RH": (14, 15, 16)}   # thigh capsule, knee sphere, foot sphere
PAIRS = {
    "c2": [(ANYMAL[a][k], ANYMAL[b][k]) for a, b in (("LF", "RF"), ("LH", "RH"), ("LF", "LH"), ("RF", "RH")) for k in range(3)]
          + [(4, 16), (8, 12), (4, 7), (8, 3)],
    "c4": [(7, 10), (8, 11), (8, 10), (11, 7), (8, 12), (11, 9), (4, 1), (6, 1), (4, 0), (6, 0), (4, 6), (2, 4), (2, 6)],
}


def device_info():
    name = torch.cuda.get_device_name(0)
    try:
        import pynvml
        pynvml.nvmlInit()
        h = pynvml.nvmlDeviceGetHandleByIndex(0)
        return name, pynvml.nvmlDeviceGetPowerManagementLimit(h) / 1000.0
    except Exception:
        return name, None


def launch_config(bt):
    """the instance the batch launches (spec 0 generic, 1 quadruped, 2 humanoid) and its warps per CTA"""
    import ctypes
    from raisimlib_b200 import capi
    L = capi.lib()
    L.rsb_internal_launch_config.argtypes = [ctypes.c_void_p] * 3
    L.rsb_internal_launch_instance.argtypes = [ctypes.c_void_p] * 3
    v = [ctypes.c_int() for _ in range(4)]
    L.rsb_internal_launch_config(bt.h, ctypes.byref(v[0]), ctypes.byref(v[1]))
    L.rsb_internal_launch_instance(bt.h, ctypes.byref(v[2]), ctypes.byref(v[3]))
    return dict(zip(("wpc", "grid", "spec", "slots"), [x.value for x in v]))


def run(key, arm, steps):
    if arm == "generic":
        os.environ["RSB_FORCE_GENERIC"] = "1"
    else:
        os.environ.pop("RSB_FORCE_GENERIC", None)
    stream = torch.cuda.current_stream()
    wl = bench.Workload(key, 0, bench.ENVS_PER_GPU)
    sim = bench.GpuSim(wl, 0, stream)
    if arm == "on":
        sim.bt.set_self_collision(PAIRS[key])
    os.environ.pop("RSB_FORCE_GENERIC", None)
    cfg = launch_config(sim.bt)
    for k in range(wl.settle + 5):
        sim.step_resident(k)
    torch.cuda.synchronize()
    k0 = wl.settle + 5
    ev = [(torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)) for _ in range(steps)]
    for k in range(steps):
        ev[k][0].record(stream)
        sim.step_resident(k0 + k)
        ev[k][1].record(stream)
    torch.cuda.synchronize()
    ms = np.array([a.elapsed_time(b) for a, b in ev])
    ct, cnt = sim.bt.contacts()
    slot = np.arange(ct.shape[1])[None, :] < cnt[:, None]
    self_ct = slot & (ct["pair_index"] < 0)
    it = sim.bt.solver_iterations()
    out = dict(config=key, arm=arm, instance=cfg, ms_per_step_median=float(np.median(ms)), ms_per_step_min=float(ms.min()),
               share_envs_with_self_contact=float(self_ct.any(1).mean()), mean_self_contacts=float(self_ct.sum(1).mean()),
               mean_contacts=float(cnt.mean()), mean_sweeps=float(it.mean()))
    del sim
    return out


def main():
    steps = int(sys.argv[1]) if len(sys.argv) > 1 else 50
    name, plimit = device_info()
    print(json.dumps({"device": name, "power_limit_w": plimit, "steps": steps}))
    for key in ("c2", "c4"):
        for arm in ("off", "generic", "on"):
            print(json.dumps(run(key, arm, steps)))


if __name__ == "__main__":
    main()
