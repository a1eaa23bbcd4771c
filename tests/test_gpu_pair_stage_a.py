"""Paired stage A of the quadruped instance (run on an H100: pytest -m gpu).

Where a CTA keeps the sub-step barrier, warps w and w ^ 4 share stage A: the leader computes both environments, lanes 16-31 the
partner's, in the partner's workspace.  Pairing decides which warp computes an environment's stage A, never what: every result must be
bit-identical to the same launches with RSB_PAIR_STAGE_A=0.  That pairing really ran is read from the stage-A clock stamps
(rsb_internal_set_profile_stage_a): lanes 0 and 16 of a leader stamp both environments with the same clock reads, which two warps
running alone do not do.
"""
import ctypes

import numpy as np
import pytest

from helpers import launch_config
from test_gpu_instances import CASES, _batch, _path

pytestmark = pytest.mark.gpu

SUBSTEPS = 4
OPTIONS = (28, 16, 14, 8, 4, 1)          # warps per CTA; the quadruped instances fit every one


def _set_stage_a_profile(capi, bt, buf):
    L = capi.lib()
    L.rsb_internal_set_profile_stage_a.argtypes = [ctypes.c_void_p, ctypes.c_void_p]
    assert L.rsb_internal_set_profile_stage_a(bt.h, ctypes.c_void_p(0 if buf is None else buf.data_ptr())) == 0


def _paired(stamps, wpc, grid):
    """environments whose stage A ran on the leader's second half-warp: all their stage-A stamps equal those of the environment of
    warp - 4 in the same CTA-round"""
    n = stamps.shape[0]
    T = wpc * grid
    e = np.arange(n)
    follower = ((e % T) % wpc & 4) != 0
    same = np.zeros(n, bool)
    idx = e[follower]
    if len(idx):
        same[idx] = (stamps[idx] == stamps[idx - 4]).all((1, 2)) & (stamps[idx] != 0).any((1, 2))
    return same


def _outputs(bt, obs):
    g, v = bt.get_state()
    rec, cnt = bt.contacts()
    return dict(obs=obs.copy(), gc=g, gv=v, contacts=rec, ncontacts=cnt, points=bt.contact_points(), iters=bt.solver_iterations(),
                resid=bt.solver_residual(), status=bt.solver_status(), tau=bt.generalized_force(), diverged=bt.diverged())


def _assert_same(runs, label):
    for k, (a, b) in enumerate(zip(*runs)):
        for key in a:
            assert a[key].shape == b[key].shape and a[key].tobytes() == b[key].tobytes(), \
                f"{label}: sample {k}: {key} differs between paired and unpaired stage A"


@pytest.mark.parametrize("key", ["c3", "c2"])
def test_bench_workloads_bit_identical(monkeypatch, key):
    """the bench's quadruped workloads at 4096 environments (two rounds of 16 warps), settled, then 12 control steps compared"""
    import torch
    import bench
    from raisimlib_b200 import capi
    assert torch.cuda.is_available(), "GPU tests need a CUDA device"
    monkeypatch.delenv("RSB_FORCE_WPC", raising=False)
    monkeypatch.delenv("RSB_SUBSTEP_BARRIER", raising=False)
    stream = torch.cuda.current_stream()
    wl = bench.Workload(key, 0, bench.ENVS_PER_GPU)
    runs, fracs = [], []
    for pair in ("1", "0"):
        monkeypatch.setenv("RSB_PAIR_STAGE_A", pair)
        sim = bench.GpuSim(wl, 0, stream)
        cfg = launch_config(capi, sim.bt)
        assert (cfg["spec"], cfg["wpc"]) == (1, 16)
        out = []
        for k in range(wl.settle + 12):
            last = k == wl.settle + 11
            if last:
                stamps = torch.zeros((bench.ENVS_PER_GPU, 4, 4), dtype=torch.int32, device="cuda")
                _set_stage_a_profile(capi, sim.bt, stamps)
            obs = sim.step_resident(k)
            if k >= wl.settle or k % 16 == 15:
                torch.cuda.synchronize()
                out.append(_outputs(sim.bt, obs.cpu().numpy()))
        _set_stage_a_profile(capi, sim.bt, None)
        fracs.append(_paired((stamps.cpu().numpy().astype(np.int64) & 0xffffffff), cfg["wpc"], cfg["grid"]).mean() * 2)
        runs.append(out)
        del sim
    print(f"{key}: environments whose stage A ran paired in the last step: {100 * fracs[0]:.1f} % (RSB_PAIR_STAGE_A=0: {100 * fracs[1]:.1f} %)")
    assert fracs[1] == 0.0
    if key == "c3":          # standing robots: most CTAs keep the sub-step barrier, and there the follower warps of both rounds are paired
        assert fracs[0] > 0.5
    assert runs[1][-1]["ncontacts"].mean() > 1.0
    _assert_same(runs, key)


def _ragged_n(wpc, grid):
    """two rounds, the last CTA of the second round partly filled; from 8 warps per CTA on with 6 warps: leaders 0 and 1 have a
    partner, leaders 2 and 3 do not"""
    T = wpc * grid
    return T + 3 * wpc + (6 if wpc >= 8 else wpc // 2)


@pytest.mark.parametrize("name", ["anymal", "quad_feet"])
def test_every_cta_size_ragged_round_wrench_limits(capi_mod, monkeypatch, name):
    """every CTA size, a ragged last round (a leader without a partner), stiff PD targets driving joints past their stops and actuators
    to their effort limits, an external wrench on every environment (the leader applies its partner's row): 10 control steps"""
    import torch
    capi = capi_mod
    monkeypatch.delenv("RSB_SUBSTEP_BARRIER", raising=False)
    monkeypatch.setenv("RSB_FORCE_WPC", "1")
    probe = capi.Batch(capi.Model(_path(CASES[name][0])), 100000)
    sms = launch_config(capi, probe)["grid"]
    del probe
    for wpc in OPTIONS:
        grid = 2 * sms if wpc == 14 else sms
        n = _ragged_n(wpc, grid)
        runs, paired = [], []
        for pair in ("1", "0"):
            monkeypatch.setenv("RSB_PAIR_STAGE_A", pair)
            t, bt, o64, o32, gc, gv, kp, kd, pt, cfg = _batch(capi, monkeypatch, name, n, "hm", seed=3000 + wpc, wpc=wpc)
            assert cfg["wpc"] == wpc and cfg["grid"] == grid
            rng = np.random.default_rng(11)
            obs = np.empty((n, bt.ob_dim()), np.float32)
            out = []
            limit_rows = effort = 0
            for k in range(10):
                body = 1 + k % (t["nb"] - 1)
                bt.set_external_wrench(body, force=rng.uniform(-40, 40, (n, 3)).astype(np.float32),
                                       torque=rng.uniform(-4, 4, (n, 3)).astype(np.float32), point_body=np.float32([0.02, -0.01, 0.03]))
                tg = pt + np.float32(0.1) * rng.uniform(-1, 1, pt.shape).astype(np.float32)
                if k == 0:
                    stamps = torch.zeros((n, 4, 4), dtype=torch.int32, device="cuda")
                    _set_stage_a_profile(capi, bt, stamps)
                bt.control_step(tg, SUBSTEPS, obs)
                if k == 0:
                    _set_stage_a_profile(capi, bt, None)
                    paired.append(_paired(stamps.cpu().numpy().astype(np.int64) & 0xffffffff, wpc, grid))
                o = _outputs(bt, obs)
                lim = np.array([t["jlimit"][b] for b in range(1, t["nb"])])
                q = o["gc"][:, 7:]
                limit_rows += int(((q < lim[:, 0]) | (q > lim[:, 1])).sum())
                eff = np.array([t["jeffort"][b] for b in range(1, t["nb"])])
                effort += int((np.abs(np.abs(o["tau"][:, 6:]) - eff) < 1e-6 * eff).sum())
                out.append(o)
            runs.append(out)
            del bt
        T = wpc * grid
        e = np.arange(n)
        w = (e % T) % wpc
        last_cta = e >= T + 3 * wpc
        print(f"{name} WPC {wpc:2d} n {n}: paired {int(paired[0].sum())} followers, joints past a stop {limit_rows}, at the effort limit {effort}")
        assert limit_rows > 0 and effort > 0
        assert not paired[1].any()
        if wpc >= 8:
            # every follower warp whose leader is in the CTA-round is paired (the first launch keeps the barrier everywhere) ...
            assert paired[0][(w & 4) != 0].all()
            # ... and the ragged last CTA holds warps 0-5: followers 4, 5 paired, leaders 2, 3 alone
            assert set(w[last_cta].tolist()) == set(range(6))
        else:
            assert not paired[0].any()
        _assert_same(runs, f"{name} WPC {wpc}")


@pytest.fixture(scope="module")
def capi_mod():
    import torch
    assert torch.cuda.is_available(), "GPU tests need a CUDA device"
    from raisimlib_b200 import capi as c
    return c


def test_getters_bit_identical(capi_mod, monkeypatch):
    """integrate1() and the kinematics-only launch of the getters (they never pair: no sub-step barrier) give the same M, h, poses and
    contact records either way"""
    capi = capi_mod
    runs = []
    for pair in ("1", "0"):
        monkeypatch.setenv("RSB_PAIR_STAGE_A", pair)
        t, bt, o64, o32, gc, gv, kp, kd, pt, cfg = _batch(capi, monkeypatch, "anymal", 3001, "hm", seed=77)
        bt.set_external_wrench(3, force=np.float32([5.0, -3.0, 20.0]))
        bt.integrate1()
        out = [dict(M=bt.mass_matrix(), h=bt.nonlinearities(), R=bt.body_poses()[0], p=bt.body_poses()[1], ct=bt.contacts()[0],
                    pts=bt.contact_points())]
        bt.integrate2()
        bt.update_kinematics()
        out.append(dict(M=bt.mass_matrix(), h=bt.nonlinearities(), R=bt.body_poses()[0], p=bt.body_poses()[1], ct=bt.contacts()[0],
                        gc=bt.get_state()[0]))
        runs.append(out)
        del bt
    _assert_same(runs, "getters")
