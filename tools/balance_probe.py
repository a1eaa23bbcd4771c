#!/usr/bin/env python3
"""Where does the launch time of the bench workload go?  (run under gpurun; exploratory, not a bench value)

One environment lives in one warp and all 4096 are resident at once, so a launch ends when the slowest
environment ends.  This probe times the settled bench workload
  * as it is, with the sub-step barrier on/off,
  * with every environment replaced by a copy of the median-cost / the most expensive one (no imbalance),
  * with environments sorted by cost (K x iterations) so that similar ones share a CTA,
and prints the K / iteration histograms that explain the differences.
"""
import os, sys
import numpy as np
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
import torch
import bench
from raisimlib_b200 import capi, RSC_DIR


def setup(n):
    H, gc, gv, targets, kp, kd = bench.make_workload(0, n)
    model = capi.Model(os.path.join(RSC_DIR, "anymal_c_like.urdf"))
    bt = capi.Batch(model, n, device=0)
    bt.set_params(threshold=1e-6)
    hm = bench.HM
    bt.set_heightmap(hm["xs"], hm["ys"], hm["size"], hm["size"], 0.0, 0.0, H)
    bt.set_pd_gains(kp, kd)
    stream = torch.cuda.current_stream()
    bt.set_stream(stream.cuda_stream)
    bt.set_state(gc.astype(np.float32), gv.astype(np.float32))
    tg = torch.tensor(targets, dtype=torch.float32, device="cuda")
    vt = torch.zeros((n, 18), dtype=torch.float32, device="cuda")
    bt.set_pd_target(tg[0], vt)
    obs = torch.empty((n, bt.ob_dim()), dtype=torch.float32, device="cuda")
    return bt, tg, obs, stream


def time_launches(bt, tg, obs, stream, steps=20, k0=0, perm=None):
    ev = [(torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)) for _ in range(steps)]
    torch.cuda.synchronize()
    for k in range(steps):
        t = tg[(k0 + k) % bench.RING]
        bt.bind_pd_target(t if perm is None else t[perm].contiguous())
        ev[k][0].record(stream)
        bt.control_step(None, bench.SUBSTEPS, obs)
        ev[k][1].record(stream)
    torch.cuda.synchronize()
    ms = np.array([a.elapsed_time(b) for a, b in ev])
    return float(np.median(ms)), float(ms.min()), float(ms.max())


def stage_report(bt, tg, obs, k0, label, perm=None):
    """one launch with the in-kernel SM-clock stamps switched on"""
    import ctypes
    n = bt.n
    lib = capi.lib()
    prof = torch.zeros((n, 4, 8), dtype=torch.int32, device="cuda")
    lib.rsb_internal_set_profile.argtypes = [ctypes.c_void_p, ctypes.c_void_p]
    lib.rsb_internal_set_profile(bt.h, ctypes.c_void_p(prof.data_ptr()))
    t = tg[k0 % bench.RING]
    bt.bind_pd_target(t if perm is None else t[perm].contiguous()); bt.control_step(None, bench.SUBSTEPS, obs)
    torch.cuda.synchronize()
    lib.rsb_internal_set_profile(bt.h, ctypes.c_void_p(0))
    P = prof.cpu().numpy().astype(np.int64) & 0xffffffff
    _, cnt1 = bt.contacts(); it1 = bt.solver_iterations()
    d = lambda a, b: ((P[:, :, b] - P[:, :, a]) & 0xffffffff).astype(np.float64)
    hasD = P[:, :, 3] != 0
    tA, tB = d(0, 1), d(1, 2)
    tC = np.where(hasD, d(2, 3), d(2, 4)); tD = np.where(hasD, d(3, 4), 0.0); tE = d(4, 5)
    tot = d(0, 5)
    print("[%s] stage cycles per sub-step (mean): A %.0f  B %.0f  C %.0f  D %.0f  E %.0f  total %.0f" %
          (label, tA.mean(), tB.mean(), tC.mean(), tD.mean(), tE.mean(), tot.mean()))
    print("   A by sub-step:", [int(tA[:, k].mean()) for k in range(4)], " total by sub-step:", [int(tot[:, k].mean()) for k in range(4)])
    for name, a in (("A", tA), ("B", tB), ("C", tC), ("D", tD), ("E", tE), ("total", tot)):
        print("   %-5s p10 %.0f  p50 %.0f  p90 %.0f  p99 %.0f  max %.0f" % (name, np.quantile(a, .1), np.median(a), np.quantile(a, .9), np.quantile(a, .99), a.max()))
    return tot, tD, cnt1, it1


def main():
    n = 4096
    bt, tg, obs, stream = setup(n)
    for k in range(bench.SETTLE + 8):
        bt.bind_pd_target(tg[k % bench.RING]); bt.control_step(None, bench.SUBSTEPS, obs)
    torch.cuda.synchronize()
    gc, gv = bt.get_state()
    _, cnt = bt.contacts()
    it = bt.solver_iterations()
    print("K histogram     :", np.bincount(cnt, minlength=9).tolist())
    print("iters histogram :", np.bincount(it, minlength=8).tolist())
    cost = cnt * it
    print("K*iters mean %.2f p50 %d p90 %d p99 %d max %d" % (cost.mean(), np.median(cost), np.quantile(cost, .9), np.quantile(cost, .99), cost.max()))
    k0 = bench.SETTLE + 8

    def restore(g=gc, v=gv):
        bt.set_state(g, v)

    if "--quick" in sys.argv:
        return
    for lvl in ("1", "0"):
        os.environ["RSB_SUBSTEP_BARRIER"] = lvl
        restore()
        print("as is, barrier %s: median %.4f ms (min %.4f max %.4f)" % ((lvl,) + time_launches(bt, tg, obs, stream, k0=k0)))
    os.environ["RSB_SUBSTEP_BARRIER"] = "1"

    restore()
    tot, tD, cnt1, it1 = stage_report(bt, tg, obs, k0, "as is, barrier 1")
    wpc = 16          # pick_config's choice for 4096 quadrupeds on the 132 SMs of an H100
    ncta = (n + wpc - 1) // wpc
    pad = np.full((ncta * wpc, 4), np.nan); pad[:n] = tot
    cta = pad.reshape(ncta, wpc, 4)
    print("per CTA and sub-step: mean warp %.0f cycles, slowest warp %.0f cycles (mean over CTAs) -> imbalance factor %.2f" %
          (np.nanmean(cta), np.nanmean(np.nanmax(cta, 1)), np.nanmean(np.nanmax(cta, 1)) / np.nanmean(cta)))
    for k in range(0, 9):
        m = cnt1 == k
        if m.sum():
            print("  K=%d (%4d envs): D mean %.0f cycles/sub-step, total %.0f, iters %.2f" % (k, m.sum(), tD[m].mean(), tot[m].mean(), it1[m].mean()))
    os.environ["RSB_SUBSTEP_BARRIER"] = "0"
    restore(); stage_report(bt, tg, obs, k0, "as is, barrier 0")
    os.environ["RSB_SUBSTEP_BARRIER"] = "1"
    idx = int(np.argsort(cost, kind="stable")[n // 2])
    restore(np.tile(gc[idx], (n, 1)), np.tile(gv[idx], (n, 1)))
    stage_report(bt, tg, obs, k0, "all envs = median env, barrier 1", perm=torch.full((n,), idx, dtype=torch.long, device="cuda"))
    sms = torch.cuda.get_device_properties(0).multi_processor_count
    b2, t2, o2, s2 = setup(sms)
    b2.set_state(gc[:sms], gv[:sms])
    stage_report(b2, t2, o2, k0, "%d envs (one warp per SM)" % sms)
    b2, t2, o2, s2 = setup(sms * 4)
    b2.set_state(gc[:sms * 4], gv[:sms * 4])
    stage_report(b2, t2, o2, k0, "%d envs" % (sms * 4))

    order = np.argsort(cost, kind="stable")
    for name, idx in (("median-cost env", order[n // 2]), ("p90-cost env", order[int(n * 0.9)]), ("worst env", order[-1]), ("cheapest env", order[0])):
        g = np.tile(gc[idx], (n, 1)); v = np.tile(gv[idx], (n, 1))
        restore(g, v)
        perm = torch.full((n,), int(idx), dtype=torch.long, device="cuda")
        for lvl in ("1", "0"):
            os.environ["RSB_SUBSTEP_BARRIER"] = lvl
            restore(g, v)
            r = time_launches(bt, tg, obs, stream, steps=6, k0=k0, perm=perm)
            print("all = %-16s (K=%d iters=%d) barrier %s: first-launch-ish median %.4f ms (min %.4f max %.4f)" % ((name, cnt[idx], it[idx], lvl) + r))
    os.environ["RSB_SUBSTEP_BARRIER"] = "1"

    perm = torch.tensor(order, dtype=torch.long, device="cuda")
    restore(gc[order], gv[order])
    print("sorted by cost, barrier 1: median %.4f ms (min %.4f max %.4f)" % time_launches(bt, tg, obs, stream, k0=k0, perm=perm))
    os.environ["RSB_SUBSTEP_BARRIER"] = "0"
    restore(gc[order], gv[order])
    print("sorted by cost, barrier 0: median %.4f ms (min %.4f max %.4f)" % time_launches(bt, tg, obs, stream, k0=k0, perm=perm))
    os.environ["RSB_SUBSTEP_BARRIER"] = "1"

    # fewer environments than warp slots: how does the launch time fall with the resident count?
    for m in (2048, 1024, 512, sms):
        b2, t2, o2, s2 = setup(m)
        b2.set_state(gc[:m], gv[:m])
        r = time_launches(b2, t2, o2, s2, k0=k0)
        print("n = %4d envs: median %.4f ms -> %.3e env-steps/s" % (m, r[0], m * bench.SUBSTEPS / r[0] * 1e3))
    for m in (8192, 16384):
        b2, t2, o2, s2 = setup(m)
        for k in range(bench.SETTLE + 8):
            b2.bind_pd_target(t2[k % bench.RING]); b2.control_step(None, bench.SUBSTEPS, o2)
        r = time_launches(b2, t2, o2, s2, k0=k0)
        print("n = %5d envs (settled): median %.4f ms -> %.3e env-steps/s" % (m, r[0], m * bench.SUBSTEPS / r[0] * 1e3))


if __name__ == "__main__":
    main()
