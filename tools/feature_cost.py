#!/usr/bin/env python3
"""What a feature of the batched step costs: each of the feature's modes timed in one process, alternating.

    python tools/feature_cost.py FEATURE [--parent-lib PATH] [--configs c3,c4] [--envs N] [--steps K] [--warmup W] [--repeats R]
                                 [--out FILE.json]
    python tools/feature_cost.py --list

For every config (bench.py's BASELINE configs: c2, c3, c4) each mode builds its batch or batches on the same seeded workload and
settles them before anything is timed; then every mode is warmed up and timed --repeats times, alternating with the others.  One
iteration is one control step, or one call for the getter and terrain modes.  It is timed with a CUDA event pair on the batch's stream,
L2 evicted before each iteration as bench.py does; terrain_curriculum takes the host wall time per call instead, since each of its
calls waits for its device check and that is what the caller pays.  Per mode the output has the median of the runs' medians, the runs,
their spread ((max - min) / median) and the kernel launches per iteration; for features with one batch per mode also whether each
mode's final state equals the reference mode's bit for bit.  --parent-lib PATH adds the mode `parent` first: the feature's first mode on
a batch of another build of the library (the commit before the feature), loaded beside this one.  The card's name, power limit and SM
clock are read in the same run.  JSON goes to stdout and to --out.
"""
import argparse
import importlib.util
import itertools
import json
import os
import subprocess
import sys
import time

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

import torch  # noqa: E402
import raisimlib_b200  # noqa: E402
from raisimlib_b200 import capi, RSC_DIR  # noqa: E402
from bench import GC0, HM, L2_FLUSH_BYTES, SUBSTEPS, GpuSim, Workload  # noqa: E402

FEET = ["LF_FOOT", "RF_FOOT", "LH_FOOT", "RH_FOOT"]
FRAMES = ["base"] + FEET
HISTORY, LAYERS, WIDTH = 3, 3, 32        # the actuator network's shape
MAPS = 16                                # maps in the terrain curriculum's atlas


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


def make_sim(wl, binding):
    raisimlib_b200.capi = binding           # GpuSim takes the binding from the package
    try:
        return GpuSim(wl, 0, torch.cuda.current_stream())
    finally:
        raisimlib_b200.capi = capi


def control_steps(sim, k0, after=None):
    """one control step per call, continuing the workload's control ring from step k0, then `after()`"""
    k = itertools.count(k0)

    def run():
        sim.step_resident(next(k))
        if after:
            after()
    return run


def per_mode(prepare):
    """set-up of a feature with one batch per mode: bench.py's batch of the config, `prepare(bt, mode, wl)` turns the mode on (and may
    return a call to make after every timed step), then the workload's settling steps"""
    def setup(wl, binding, modes):
        out = {}
        for m in modes:
            sim = make_sim(wl, binding)
            after = prepare(sim.bt, m, wl)
            for k in range(wl.settle):
                sim.step_resident(k)
            out[m] = (control_steps(sim, wl.settle, after), sim.bt)
        return out
    return setup


# ---------------------------------------------------------------- features with one batch per mode
def contact_forces(bt, mode, wl):
    """rsb_batch_set_contact_bodies: the 4 feet, all 13 bodies, or all 13 read into torch CUDA tensors after every step"""
    if mode == "feet":
        bt.set_contact_bodies_by_name(FEET)
    elif mode.startswith("all"):
        bt.set_contact_bodies(list(range(13)))
    if mode == "all+read":
        force, steps = torch.empty((wl.n, 13, 3), device="cuda"), torch.empty((wl.n, 13), dtype=torch.int32, device="cuda")
        return lambda: bt.body_contact_forces_into(force, steps)


def contact_force_summary(batches):
    f, s = batches["all"].body_contact_forces()
    return {"mean_bodies_in_contact": float((s > 0).sum(1).mean()), "mean_total_force_z": float(f[:, :, 2].sum(1).mean())}


def body_inertia(bt, mode, wl):
    """rsb_batch_set_body_inertia: a distinct row in every environment, the model's values x U(0.98, 1.02) so the robots still stand"""
    if mode == "rows":
        rows = np.tile(bt.model_body_inertia(), (wl.n, 1, 1))
        scale = np.random.default_rng(1).uniform(0.98, 1.02, (wl.n, rows.shape[1], 1)).astype(np.float32)
        rows[:, :, :1] *= scale
        rows[:, :, 4:] *= scale
        bt.set_body_inertia(rows)


def contact_friction(bt, mode, wl):
    """rsb_batch_set_contact_friction: rows at the batch-level value (params.mu on every collision body), so the physics is bit for bit
    that of `none` and the difference is the load of the row entry per contact alone"""
    if mode == "rows":
        bt.set_contact_friction(np.full((wl.n, bt.model.ncoll), bt.get_params().mu, np.float32))


def batch_value_rows(bt, wl, n):
    """[n, nv, 3]: the workload's gains and the model's effort limits, in the batch's gv order"""
    t = bt.model.tables()
    row = np.zeros((bt.nv, 3), np.float32)
    row[:, 0], row[:, 1] = wl.kp, wl.kd
    row[:, 2] = 3.0e38
    for b in range(1, t["nb"]):
        row[t["vidx"][b], 2] = min(t["jeffort"][b], 3.0e38)
    return np.tile(row, (n, 1, 1))


def actuator_params(bt, mode, wl):
    """rsb_batch_set_actuator_params: rows at the batch-level values, so the physics is bit for bit that of `none` and the difference is
    the load of three row entries per dof and sub-step alone"""
    if mode == "rows":
        bt.set_actuator_params(batch_value_rows(bt, wl, wl.n))


def zero_output_network(rng):
    """[(W, b)]: dense random hidden layers, zero output layer (net = 0 exactly)"""
    out, nin = [], 2 * HISTORY
    for _ in range(LAYERS):
        out.append((rng.uniform(-1, 1, (WIDTH, nin)) / np.sqrt(nin), rng.uniform(-0.3, 0.3, WIDTH)))
        nin = WIDTH
    out.append((np.zeros((1, WIDTH)), np.zeros(1)))
    return [(w.astype(np.float32), b.astype(np.float32)) for w, b in out]


def actuator_network(bt, mode, wl):
    """`pd` the PD law; `limp` kp = kd = 0 rows on the 12 joints, so the robots sag; `net` a network on the 12 joints whose output layer
    is zero: every weight is loaded and multiplied at every sub-step, the torque is exactly that of `limp`, so the difference between
    the two is the cost of evaluating the network"""
    if mode == "limp":
        rows = np.full((wl.n, 18, 3), -1.0, np.float32)
        rows[:, 6:, :2] = 0.0
        bt.set_actuator_params(rows)
    elif mode == "net":
        bt.set_actuator_network(list(range(6, 18)), zero_output_network(np.random.default_rng(0)), HISTORY)


def actuation_delay(bt, mode, wl):
    """rsb_batch_set_actuation_delay: every delay 0 (the delay instance of the step runs, the state equals that of `none` bit for bit),
    or delays drawn from U{0..8} sub-steps per environment"""
    if mode == "zeros":
        bt.set_actuation_delay(np.zeros(wl.n, np.int32))
    elif mode == "u0_8":
        bt.set_actuation_delay(np.random.default_rng(0).integers(0, 9, wl.n).astype(np.int32))


# ---------------------------------------------------------------- features whose modes share batches
def frame_kinematics(wl, binding, modes):
    """frames base + 4 feet on one batch, outputs into torch CUDA tensors.  `step+states` needs the kinematics pass (the poses are
    stale after a step), `step+states+jac` does not; the kernel-only modes run on the poses their first warm-up call made current."""
    sim = make_sim(wl, binding)
    bt, n, F = sim.bt, wl.n, len(FRAMES)
    bt.set_frames_by_name(FRAMES)
    pos, lin, ang = (torch.empty((n, F, 3), device="cuda") for _ in range(3))
    rot, jac = torch.empty((n, F, 3, 3), device="cuda"), torch.empty((n, F, 6, bt.nv), device="cuda")
    for k in range(wl.settle):
        sim.step_resident(k)
    step = control_steps(sim, wl.settle)

    def states():
        bt.frame_states_into(pos, rot, lin, ang)

    def jacobians():
        bt.frame_jacobians_into(jac)

    runs = {"step": step, "step+states": lambda: (step(), states()), "step+states+jac": lambda: (step(), states(), jacobians()),
            "kinematics": bt.update_kinematics, "states_kernel": states, "jac_kernel": jacobians}
    return {m: (runs[m], bt) for m in modes}


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


def height_scan(wl, binding, modes):
    """RaisimGym batches (rsb_batch_gym_step, 4 sub-steps per control step) on the config's height map, 30 control steps in.
    scan_base: the scan kernel alone, 187 yaw-aligned base points (legged_gym's 11 x 17 grid), poses from gc, no kinematics pass.
    scan_feet: the scan kernel alone, 52 points around each of the 4 feet; the state does not change between calls, so after the first
    warm-up call's kinematics pass each call is the scan launch only.  gym: gym_step.  gym_scan: gym_step, then the base grid's scan."""
    n, stream = wl.n, torch.cuda.current_stream()
    m = binding.Model(os.path.join(RSC_DIR, "anymal_c_like.urdf"))
    feet = [m.body_index(f) for f in FEET]
    grid, ring = base_grid(), foot_rings()
    base_pts = (np.zeros(len(grid), np.int32), grid)
    points = {"base": base_pts, "feet": (np.repeat(np.array(feet, np.int32), len(ring)), np.tile(ring, (4, 1))), "gym": base_pts}
    g = torch.Generator(device="cuda")
    g.manual_seed(7)
    acts = [0.15 * torch.randn((n, 12), device="cuda", generator=g) for _ in range(8)]
    obs, rew, done = torch.empty((n, 34), device="cuda"), torch.empty(n, device="cuda"), torch.empty(n, dtype=torch.uint8, device="cuda")

    def gym_batch(pts):
        bt = binding.Batch(m, n)
        bt.set_stream(stream.cuda_stream)
        bt.set_heightmap(HM["xs"], HM["ys"], HM["size"], HM["size"], 0.0, 0.0, wl.H)
        bt.set_params(threshold=1e-6)
        bt.set_pd_gains(np.r_[np.zeros(6), 100.0 * np.ones(12)], np.r_[np.zeros(6), 2.0 * np.ones(12)])
        g0 = GC0.copy()
        g0[2] = 0.57 + float(np.max(wl.H))
        bt.gym_configure(g0, np.zeros(18), g0[7:], 0.6 * np.ones(12), feet)
        bt.gym_reset()
        bt.set_height_scan(*pts)
        for k in range(30):
            bt.gym_step(acts[k % 8], SUBSTEPS, obs, rew, done)
        return bt

    uses = {"scan_base": "base", "scan_feet": "feet", "gym": "gym", "gym_scan": "gym"}
    bts = {b: gym_batch(points[b]) for b in dict.fromkeys(uses[md] for md in modes)}
    hb, hf = torch.empty((n, len(grid)), device="cuda"), torch.empty((n, 4 * len(ring)), device="cuda")
    k = itertools.count(30)

    def gym(scan):
        bts["gym"].gym_step(acts[next(k) % 8], SUBSTEPS, obs, rew, done)
        if scan:
            bts["gym"].height_scan_into(hb)

    runs = {"scan_base": lambda: bts["base"].height_scan_into(hb), "scan_feet": lambda: bts["feet"].height_scan_into(hf),
            "gym": lambda: gym(False), "gym_scan": lambda: gym(True)}
    return {md: (runs[md], bts[uses[md]]) for md in modes}


def terrain_curriculum(wl, binding, modes):
    """calls on an atlas of 16 random maps of bench.py's 513 x 513 size (the config gives the number of environments only):
    index_host / index_device: rsb_batch_set_heightmap_index of all environments from a pageable numpy array / a torch CUDA tensor;
    update_host / update_device: rsb_batch_update_heightmaps of one map, likewise; atlas_16: for comparison, the route without these
    calls, rsb_batch_set_heightmaps of the whole atlas and index"""
    n = wl.n
    rng = np.random.default_rng(3)
    H = rng.uniform(-0.1, 0.1, (MAPS, HM["ys"], HM["xs"])).astype(np.float32)
    idx = [rng.integers(0, MAPS, n).astype(np.int32) for _ in range(4)]
    didx = [torch.from_numpy(x).cuda() for x in idx]
    one, one_dev = H[3:4].copy(), torch.from_numpy(H[3:4]).cuda()
    bt = binding.Batch(binding.Model(os.path.join(RSC_DIR, "anymal_c_like.urdf")), n)
    bt.set_stream(torch.cuda.current_stream().cuda_stream)
    bt.set_heightmaps(HM["size"], HM["size"], 0.0, 0.0, H, idx[0])
    calls = {"index_host": lambda k: bt.set_heightmap_index(idx[k % 4]), "index_device": lambda k: bt.set_heightmap_index_from(didx[k % 4]),
             "update_host": lambda k: bt.update_heightmaps(3, one), "update_device": lambda k: bt.update_heightmaps_from(3, one_dev),
             "atlas_16": lambda k: bt.set_heightmaps(HM["size"], HM["size"], 0.0, 0.0, H, idx[k % 4])}
    k = itertools.count(1)
    return {m: ((lambda c=calls[m]: c(next(k))), bt) for m in modes}


# Per feature: its default configs, its modes in order, the set-up that gives every mode (its one timed iteration, the batch it runs
# on); with one batch per mode, `ref` is the mode whose final state every other one is compared with.
FEATURES = {
    "contact_forces": dict(configs="c3,c2", modes=["none", "feet", "all", "all+read"], setup=per_mode(contact_forces), ref="none",
                           summary=contact_force_summary),
    "body_inertia": dict(configs="c3,c4", modes=["none", "rows"], setup=per_mode(body_inertia), ref="none"),
    "contact_friction": dict(configs="c3", modes=["none", "rows"], setup=per_mode(contact_friction), ref="none"),
    "actuator_params": dict(configs="c3", modes=["none", "rows"], setup=per_mode(actuator_params), ref="none"),
    "actuator_network": dict(configs="c3", modes=["pd", "limp", "net"], setup=per_mode(actuator_network), ref="limp",
                             summary=lambda batches: {"network": dict(dofs=12, history=HISTORY, layers=LAYERS, width=WIDTH)}),
    "actuation_delay": dict(configs="c3,c4", modes=["none", "zeros", "u0_8"], setup=per_mode(actuation_delay), ref="none"),
    "frame_kinematics": dict(configs="c3", modes=["step", "step+states", "step+states+jac", "kinematics", "states_kernel", "jac_kernel"],
                             setup=frame_kinematics),
    "height_scan": dict(configs="c3", modes=["scan_base", "scan_feet", "gym", "gym_scan"], setup=height_scan),
    "terrain_curriculum": dict(configs="c3", modes=["index_host", "index_device", "update_host", "update_device", "atlas_16"],
                               setup=terrain_curriculum, host_timed=True),
}


def main():
    ap = argparse.ArgumentParser(description="What a feature of the batched step costs, its modes alternated in one process")
    ap.add_argument("feature", nargs="?", choices=FEATURES)
    ap.add_argument("--list", action="store_true", help="print every feature with its default configs and its modes")
    ap.add_argument("--parent-lib", help="another build of librsb.so: mode `parent` runs the feature's first mode on it")
    ap.add_argument("--configs", help="comma-separated bench.py configs (default: the feature's)")
    ap.add_argument("--envs", type=int, default=4096)
    ap.add_argument("--steps", type=int, default=200, help="timed iterations per run")
    ap.add_argument("--warmup", type=int, default=20, help="untimed iterations before every run")
    ap.add_argument("--repeats", type=int, default=5, help="runs of every mode, alternated")
    ap.add_argument("--out", help="also write the JSON result here")
    args = ap.parse_args()
    if args.list:
        for name, f in FEATURES.items():
            print(f"{name:20s} configs {f['configs']:7s} modes {' '.join(f['modes'])}")
        return
    if not args.feature:
        ap.error("name a feature (--list shows them)")
    if not torch.cuda.is_available():
        raise SystemExit("feature_cost.py needs a CUDA device")
    f = FEATURES[args.feature]
    host = f.get("host_timed", False)
    parent = load_capi(os.path.abspath(args.parent_lib)) if args.parent_lib else None
    stream = torch.cuda.current_stream()
    flush = torch.empty(L2_FLUSH_BYTES // 4, dtype=torch.float32, device="cuda")

    def timed(run, bt):
        """median ms per iteration over --steps iterations, and kernel launches per iteration"""
        for _ in range(args.warmup):
            run()
        ev = [] if host else [(torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)) for _ in range(args.steps)]
        t = []
        torch.cuda.synchronize()
        l0 = bt.launch_count()
        for k in range(args.steps):
            if host:
                t0 = time.perf_counter()
                run()
                t.append(1e3 * (time.perf_counter() - t0))
            else:
                flush.fill_(float(k))
                ev[k][0].record(stream)
                run()
                ev[k][1].record(stream)
        torch.cuda.synchronize()
        if not host:
            t = [a.elapsed_time(b) for a, b in ev]
        return float(np.median(t)), (bt.launch_count() - l0) / args.steps

    def measure(key):
        wl = Workload(key, 0, args.envs)
        modes = {}
        if parent:
            modes["parent"] = f["setup"](wl, parent, f["modes"][:1])[f["modes"][0]]
        modes.update(f["setup"](wl, capi, f["modes"]))
        runs, launches = {m: [] for m in modes}, {}
        for _ in range(args.repeats):
            for m, (run, bt) in modes.items():
                ms, launches[m] = timed(run, bt)
                runs[m].append(ms)
        med = {m: float(np.median(v)) for m, v in runs.items()}
        res = dict(workload=wl.name, median_ms=med, runs_ms=runs, spread={m: (max(v) - min(v)) / med[m] for m, v in runs.items()},
                   launches_per_iteration=launches)
        if "ref" in f:
            ref = modes[f["ref"]][1].get_state()[0].tobytes()
            res["state_equal_to_" + f["ref"]] = {m: bt.get_state()[0].tobytes() == ref for m, (_, bt) in modes.items()}
        if "summary" in f:
            res.update(f["summary"]({m: bt for m, (_, bt) in modes.items()}))
        base = f["modes"][0]
        print(f"--- {key}: {wl.name}")
        for m in modes:
            same = f"; state equal to {f['ref']} {res['state_equal_to_' + f['ref']][m]}" if "ref" in f else ""
            print(f"{m:16s} {med[m]:.4f} ms  ({100 * (med[m] / med[base] - 1):+.2f} % vs {base}; runs {', '.join(f'{x:.4f}' for x in runs[m])}; "
                  f"spread {100 * res['spread'][m]:.2f} %; launches {launches[m]:.2f}{same})")
        return res

    res = {"feature": args.feature, "device": torch.cuda.get_device_name(0), "parent_lib": args.parent_lib, "envs": args.envs,
           "steps": args.steps, "warmup": args.warmup, "repeats": args.repeats,
           "timing": "host wall time per call" if host else "CUDA events per iteration, L2 evicted before each",
           "configs": {key: measure(key) for key in (args.configs or f["configs"]).split(",")}}
    res["nvidia_smi"] = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm,clocks.sm", "--format=csv,noheader", "-i", "0"],
                                       capture_output=True, text=True).stdout.strip()
    print(res["nvidia_smi"])
    print(json.dumps(res))
    if args.out:
        with open(args.out, "w") as fh:
            json.dump(res, fh, indent=1)


if __name__ == "__main__":
    main()
