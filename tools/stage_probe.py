#!/usr/bin/env python3
"""In-kernel stage timers for any bench workload (run under gpurun; exploratory, never a bench value).

usage: stage_probe.py c3|c2|c4 [n_envs] -- prints cycles per sub-step of one environment in stages A..E (SM-clock stamps written by the
step kernel through rsb_internal_set_profile), launch times with the sub-step barrier on / off, the sweep / contact histograms, and
what the slowest warp of each CTA-round costs behind the sub-step barrier; for the quadruped instance also the split of stage A
(RSB_PAIR_STAGE_A=0 runs it unpaired)."""
import ctypes, os, sys
import numpy as np
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
import torch
import bench
from raisimlib_b200 import capi


def launch_ms(sim, k0, steps=12):
    stream = torch.cuda.current_stream()
    ev = [(torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)) for _ in range(steps)]
    torch.cuda.synchronize()
    for k in range(steps):
        ev[k][0].record(stream); sim.step_resident(k0 + k); ev[k][1].record(stream)
    torch.cuda.synchronize()
    ms = np.array([a.elapsed_time(b) for a, b in ev])
    return float(np.median(ms)), float(ms.min()), float(ms.max())


def main():
    key = sys.argv[1] if len(sys.argv) > 1 else "c3"
    n = int(sys.argv[2]) if len(sys.argv) > 2 else bench.ENVS_PER_GPU
    stream = torch.cuda.current_stream()
    wl = bench.Workload(key, 0, n)
    sim = bench.GpuSim(wl, 0, stream)
    if os.environ.get("RSB_PROBE_CONTACT_BODIES"):     # e.g. 3,6,9,12: per-body contact forces on (their cost shows in stage E)
        sim.bt.set_contact_bodies([int(x) for x in os.environ["RSB_PROBE_CONTACT_BODIES"].split(",")])
    if os.environ.get("RSB_PROBE_BODY_INERTIA"):       # 1: a distinct inertial row in every environment (their cost shows in stage A)
        rows = np.tile(sim.bt.model_body_inertia(), (n, 1, 1))
        rows[:, :, :1] *= np.random.default_rng(1).uniform(0.98, 1.02, (n, rows.shape[1], 1)).astype(np.float32)
        sim.bt.set_body_inertia(rows)
    for k in range(wl.settle + 8):
        sim.step_resident(k)
    torch.cuda.synchronize()
    k0 = wl.settle + 8
    g, v = sim.bt.get_state()
    st = sim.stats()
    print(key, wl.name)
    print("  K hist", st["contacts_histogram"], "sweeps", st["sweeps_histogram"], "mean %.2f max %d" % (st["mean_solver_sweeps"], st["max_solver_sweeps"]))
    ref = None
    for lvl in os.environ.get("RSB_PROBE_LEVELS", "1,0").split(","):
        os.environ["RSB_SUBSTEP_BARRIER"] = lvl
        sim.bt.set_state(g, v)
        t = launch_ms(sim, k0)
        ge, ve = sim.bt.get_state()
        if ref is None:
            ref = (ge, ve)
        same = bool((ge == ref[0]).all() and (ve == ref[1]).all())      # the alignment mode must not change a single bit of the result
        print("  barrier %s: launch median %.4f ms (min %.4f max %.4f) -> %.3e env-steps/s   state identical to the first mode: %s"
              % ((lvl,) + t + (n * bench.SUBSTEPS / t[0] * 1e3, same)))
    os.environ.pop("RSB_SUBSTEP_BARRIER")
    if os.environ.get("RSB_PROBE_STAGE_LEVEL"):       # stage timers under this alignment mode instead of the default
        os.environ["RSB_SUBSTEP_BARRIER"] = os.environ["RSB_PROBE_STAGE_LEVEL"]
    lib = capi.lib()
    lib.rsb_internal_set_profile.argtypes = [ctypes.c_void_p, ctypes.c_void_p]
    lib.rsb_internal_launch_config.argtypes = [ctypes.c_void_p] * 3
    wpc, grid = ctypes.c_int(), ctypes.c_int()
    lib.rsb_internal_launch_config(sim.bt.h, ctypes.byref(wpc), ctypes.byref(grid))
    wpc, grid = wpc.value, grid.value
    lib.rsb_internal_set_profile_stage_a.argtypes = [ctypes.c_void_p, ctypes.c_void_p]
    sim.bt.set_state(g, v)
    prof = torch.zeros((n, 4, 8), dtype=torch.int32, device="cuda")
    prof_a = torch.zeros((n, 4, 4), dtype=torch.int32, device="cuda")      # quadruped instance: stamps inside stage A
    lib.rsb_internal_set_profile(sim.bt.h, ctypes.c_void_p(prof.data_ptr()))
    lib.rsb_internal_set_profile_stage_a(sim.bt.h, ctypes.c_void_p(prof_a.data_ptr()))
    sim.step_resident(k0)
    torch.cuda.synchronize()
    lib.rsb_internal_set_profile(sim.bt.h, ctypes.c_void_p(0))
    lib.rsb_internal_set_profile_stage_a(sim.bt.h, ctypes.c_void_p(0))
    P = prof.cpu().numpy().astype(np.int64) & 0xffffffff
    d = lambda a, b: ((P[:, :, b] - P[:, :, a]) & 0xffffffff).astype(np.float64)
    PA = prof_a.cpu().numpy().astype(np.int64) & 0xffffffff
    if (PA != 0).any():
        # stage A from the environment's own start stamp: FK walk | per-body terms | subtree sums | M columns | to the end of stage A
        # (a paired environment's last part is the wait for the pair barrier, an unpaired one's the stage-A prof stamp)
        S = np.concatenate([P[:, :, :1], PA, P[:, :, 1:2]], axis=2)
        parts = [((S[:, :, i + 1] - S[:, :, i]) & 0xffffffff).astype(np.float64) for i in range(5)]
        print("  stage A split (cycles per sub-step):")
        for name, a in zip(("FK walk", "per-body terms", "subtree sums", "M columns", "to the end"), parts):
            print("     %-14s mean %.0f  p10 %.0f  p50 %.0f  p90 %.0f  max %.0f" % (name, a.mean(), np.quantile(a, .1), np.median(a), np.quantile(a, .9), a.max()))
    hasD = P[:, :, 3] != 0
    tA, tB = d(0, 1), d(1, 2)
    tC = np.where(hasD, d(2, 3), d(2, 4)); tD = np.where(hasD, d(3, 4), 0.0); tE = d(4, 5); tot = d(0, 5)
    print("  stage cycles per sub-step (mean): A %.0f  B %.0f  C %.0f  D %.0f  E %.0f  total %.0f" % (tA.mean(), tB.mean(), tC.mean(), tD.mean(), tE.mean(), tot.mean()))
    for name, a in (("A", tA), ("B", tB), ("C", tC), ("D", tD), ("E", tE), ("total", tot)):
        print("     %-5s p10 %.0f  p50 %.0f  p90 %.0f  p99 %.0f  max %.0f" % (name, np.quantile(a, .1), np.median(a), np.quantile(a, .9), np.quantile(a, .99), a.max()))
    if (P[:, :, 6] != 0).any():      # inner stamps of stage B: candidate loop | sphere groups + compaction
        print("  stage B split: candidates + sphere groups %.0f  selection + contact records %.0f  | penetrating candidates: mean %.2f max %d" % (d(1, 6).mean(), d(6, 2).mean(), P[:, :, 7].mean(), P[:, :, 7].max()))
    it = sim.bt.solver_iterations(); _, cnt = sim.bt.contacts()
    upd = np.maximum(1, it * cnt)
    print("  D cycles per contact update (last sub-step): median %.0f" % np.median(tD[:, 3] / upd))
    # behind the sub-step barrier a CTA-round (the warps of one CTA in one round) lasts, per sub-step, as long as its slowest warp:
    # sum over the sub-steps of the group maximum against the mean busy time (the stamps exclude the barrier wait)
    T = wpc * grid
    e = np.arange(n)
    group = (e // T) * grid + (e % T) // wpc
    gmax = np.zeros((group.max() + 1, tot.shape[1]))
    np.maximum.at(gmax, group, tot)
    print("  CTA-rounds (%d warps x %d CTAs, %d environments per round): mean of the per-sub-step group max %.0f cycles per launch, "
          "mean busy %.0f (%.2fx)" % (wpc, grid, T, gmax.sum(1).mean(), tot.sum(1).mean(), gmax.sum(1).mean() / tot.sum(1).mean()))


if __name__ == "__main__":
    main()
