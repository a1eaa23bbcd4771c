"""Per-environment PD gains and actuator effort limits (rsb_batch_set_actuator_params / rsb_batch_clear_actuator_params) through the
C-ABI on an H100 (pytest -m gpu): bit-identity with the batch-level gains and URDF limits on every compiled instance in both control
modes, every environment against a float64 oracle configured with that environment's gains and limits, an analytic pendulum, batch-level
resolution and persistence, the fused gym task, launch shapes, and the rules of the contract (sources, refusals, launch count, the C++
facade)."""
import ctypes as C
import os
import subprocess

import numpy as np
import pytest

from conftest import ROOT, RSC
from helpers import ANYMAL_GC0, THRESH, effort_limits, setup_batch
from oracle.oracle import Oracle
from test_gpu_contact_forces import _make, _outputs, _same
from test_self_collision_oracle import anymal_leg_pairs

pytestmark = pytest.mark.gpu

SUB, DT = 4, 0.0025


@pytest.fixture(scope="module")
def capi():
    import torch
    assert torch.cuda.is_available(), "GPU tests need a CUDA device"
    from raisimlib_b200 import capi as c
    return c


# name -> (case of test_gpu_contact_forces, terrain, self-collision pairs)
SETUPS = {"quadruped_hm": ("quadruped", "hm", False), "humanoid_ground": ("humanoid", "ground", False), "generic_self": ("generic", "hm", True)}
MODES = ("pd", "force")


_limits = effort_limits


def _setup(capi, monkeypatch, which, n, seed, mode="pd", wpc=None):
    """_make's robots with targets (PD) or feed-forward torques (force) far enough away that some joints saturate at their URDF limit;
    the leg pairs on the generic instance"""
    case, terrain, pairs = SETUPS[which]
    c = _make(capi, monkeypatch, case, n, terrain, seed, wpc=wpc, oracles=False)
    t, bt = c["t"], c["bt"]
    rng = np.random.default_rng(seed + 1)
    if mode == "pd":
        pt = c["pt"].copy(); pt[:, 7:] += rng.uniform(-0.4, 0.4, (n, t["nq"] - 7)).astype(np.float32)
        bt.set_pd_target(pt, np.zeros((n, t["nv"]), np.float32))
    else:
        bt.set_control_mode(capi.FORCE_AND_TORQUE)
        tau = np.zeros((n, t["nv"]), np.float32); tau[:, 6:] = rng.uniform(-1.3, 1.3, (n, t["nv"] - 6)) * np.minimum(_limits(t)[6:], 200.0)
        bt.set_generalized_force(tau)
    if pairs:
        bt.set_self_collision(anymal_leg_pairs())
    return c


def _random_rows(t, n, seed):
    """a different row in every environment: kp in [50, 600], kd in [0.5, 10], the effort limit in [0.1, 1.2] x the URDF's; some exact
    0, some -1, some effort +inf"""
    rng = np.random.default_rng(seed)
    nv = t["nv"]
    rows = np.empty((n, nv, 3))
    rows[:, :, 0] = rng.uniform(50.0, 600.0, (n, nv))
    rows[:, :, 1] = rng.uniform(0.5, 10.0, (n, nv))
    rows[:, :, 2] = rng.uniform(0.1, 1.2, (n, nv)) * np.minimum(_limits(t), 300.0)
    rows[rng.random((n, nv, 3)) < 0.05] = 0.0
    rows[rng.random((n, nv, 3)) < 0.15] = -1.0
    rows[:, :, 2][rng.random((n, nv)) < 0.05] = np.inf
    return rows.astype(np.float32)


def _batch_values(c):
    """the row every environment resolves to without rows: _make's gains, the URDF's effort limits"""
    row = np.stack([c["kp"], c["kd"], _limits(c["t"])], axis=1)
    return np.tile(row, (c["n"], 1, 1)).astype(np.float32)


def _all_outputs(bt):
    o = _outputs(bt)
    f, s = bt.body_contact_forces()
    o.update(f=f, s=s)
    return o


# ---- 1: bit-identity with the batch-level gains and limits ---------------------------------------------------------------------------

@pytest.mark.parametrize("mode", MODES)
@pytest.mark.parametrize("which", list(SETUPS))
def test_no_rows_minus_one_reset_cleared_and_batch_values_agree(capi, monkeypatch, which, mode):
    """no rows, rows of -1, rows reset with NULL, rows set then cleared, and rows equal to the batch-level values: every output of 8
    control steps bit for bit, including the generalized force and the per-body contact forces, with joints at their effort limit"""
    n = 300
    runs = {}
    for rmode in ("never", "minus_one", "null_reset", "cleared", "batch_values"):
        c = _setup(capi, monkeypatch, which, n, seed=81, mode=mode)
        bt, t = c["bt"], c["t"]
        bt.set_contact_bodies(list(range(min(t["nb"], 32))))
        if rmode == "minus_one":
            bt.set_actuator_params(np.full((n, t["nv"], 3), -1.0, np.float32))
        elif rmode == "null_reset":
            bt.set_actuator_params(_random_rows(t, n, 3))
            bt.set_actuator_params(None)
        elif rmode == "cleared":
            bt.set_actuator_params(_random_rows(t, n, 3))
            bt.integrate(SUB); bt.set_state(c["gc"], c["gv"])
            bt.clear_actuator_params()
        elif rmode == "batch_values":
            bt.set_actuator_params(_batch_values(c))
        runs[rmode] = []
        for k in range(8):
            bt.integrate(SUB)
            runs[rmode].append(_all_outputs(bt))
    lim = _limits(c["t"])
    saturated = sum(int((np.abs(np.abs(r["tau"][:, 6:]) - lim[6:]) < 1e-3 * lim[6:]).sum()) for r in runs["never"])
    contacts = sum(int(r["cnt"].sum()) for r in runs["never"])
    print(f"{which} {mode}: {saturated} dof-steps at the effort limit, {contacts} contacts over the 8 control steps")
    assert saturated > 100 and contacts > n
    for rmode in runs:
        for k in range(8):
            _same(runs["never"][k], runs[rmode][k], f"{which} {mode} {rmode}, control step {k}: ")


def test_unlimited_and_base_entries_store_the_batch_values(capi, monkeypatch):
    """effort +inf and effort 3e38 (the blob's "none") compute the same bits, and so do any values in the base dofs' entries and -1"""
    n = 200
    out = {}
    for mode in ("inf", "none_value", "base_garbage"):
        c = _setup(capi, monkeypatch, "quadruped_hm", n, seed=83)
        rows = _random_rows(c["t"], n, 17)
        rows[:, :6] = -1.0
        rows[:, 6:12, 2] = {"inf": np.inf, "none_value": 3.0e38, "base_garbage": np.inf}[mode]
        if mode == "base_garbage":
            rows[:, :6] = np.random.default_rng(3).uniform(0.0, 1e4, (n, 6, 3))
        c["bt"].set_actuator_params(rows)
        for k in range(4):
            c["bt"].integrate(SUB)
        out[mode] = _outputs(c["bt"])
    _same(out["inf"], out["none_value"], "effort +inf against 3e38: ")
    _same(out["inf"], out["base_garbage"], "base entries: ")


# ---- 2: against the oracle -----------------------------------------------------------------------------------------------------------

def test_every_environment_matches_an_oracle_with_its_gains_and_limits(capi):
    """256 quadrupeds, every one with its own kp, kd (some 0, some -1 on top of batch-level gains) and effort limits (some saturating,
    some -1, some 0, some +inf), against one float64 oracle per environment built with those limits and stepped with those gains: the
    bounds of test_actuator_effort_limits_match_oracle"""
    n = 256
    t, bt, _, _, gc, gv, _ = setup_batch(capi, "anymal_c_like.urdf", n, seed=191, base_z=0.62, vel=0.2, tau_scale=0.0, joint_scale=0.2)
    rng = np.random.default_rng(192)
    kp_b = np.r_[np.zeros(6), 800.0 * np.ones(12)]; kd_b = np.r_[np.zeros(6), 10.0 * np.ones(12)]
    rows = np.empty((n, 18, 3))
    rows[:, :, 0] = rng.uniform(100.0, 2000.0, (n, 18)); rows[:, :, 1] = rng.uniform(1.0, 20.0, (n, 18))
    rows[:, :, 2] = rng.uniform(20.0, 80.0, (n, 18))
    rows[:, :, :2][rng.random((n, 18, 2)) < 0.05] = 0.0
    rows[rng.random((n, 18, 3)) < 0.15] = -1.0
    rows[:, :, 2][rng.random((n, 18)) < 0.03] = 0.0
    rows[:, :, 2][rng.random((n, 18)) < 0.03] = np.inf
    rows = rows.astype(np.float32)
    pt = gc.copy(); pt[:, 7:] += rng.uniform(-0.6, 0.6, (n, 12))
    pt32, vt = pt.astype(np.float32), np.zeros((n, 18))
    bt.set_control_mode(capi.PD_PLUS_FEEDFORWARD_TORQUE)
    bt.set_pd_gains(kp_b, kd_b)
    bt.set_pd_target(pt32, vt.astype(np.float32))
    bt.set_actuator_params(rows)
    r = rows.astype(np.float64)
    kp = np.where(r[:, :, 0] >= 0, r[:, :, 0], kp_b); kd = np.where(r[:, :, 1] >= 0, r[:, :, 1], kd_b)
    kp[:, :6] = 0.0; kd[:, :6] = 0.0
    lim = np.where(r[:, :, 2] >= 0, r[:, :, 2], _limits(t))
    oracles = []
    for e in range(n):
        jeff = t["jeffort"].copy()
        for b in range(1, t["nb"]):
            jeff[b] = lim[e, t["vidx"][b]]
        o = Oracle(dict(t, jeffort=jeff), params=dict(threshold=THRESH))
        o.set_ground(0.0)
        oracles.append(o)
    a, b_ = gc.copy(), gv.copy()
    status, tau_ref = np.zeros(n, np.int32), np.zeros((n, 18))
    for k in range(20):
        bt.integrate(1)
        ta = bt.generalized_force() if k == 0 else None
        for e in range(n):
            ae, be = a[e:e + 1].copy(), b_[e:e + 1].copy()
            d = oracles[e].step(ae, be, ptarget=pt32[e:e + 1].astype(np.float64), vtarget=vt[e:e + 1], kp=kp[e], kd=kd[e], debug=True)
            a[e], b_[e] = ae[0], be[0]
            status[e] = d["status"][0]
            if k == 0:
                tau_ref[e] = d["tau_applied"][0]
        if k == 0:
            sat_ref = np.abs(np.abs(tau_ref[:, 6:]) - lim[:, 6:]) < 1e-9
            sat_gpu = np.abs(np.abs(ta[:, 6:]) - lim[:, 6:]) < 1e-4
            print(f"step 0: {int(sat_ref.sum())} of {sat_ref.size} joint dofs at their own limit; sets agree on {100 * (sat_ref == sat_gpu).mean():.3f} %")
            assert sat_ref.mean() > 0.2 and (sat_ref == sat_gpu).mean() > 0.999
    g, v = bt.get_state()
    conv = (bt.solver_status() <= 1) & (status <= 1)
    eg = np.abs(g - a).max(1)[conv]
    print(f"per-environment gains and limits, 20 steps ({int(conv.sum())} converged): median |dgc| {np.median(eg):.2e} p90 {np.quantile(eg, 0.9):.2e}")
    assert conv.mean() > 0.8
    assert np.median(eg) < 2e-5 and np.quantile(eg, 0.9) < 2e-4


# ---- 3: analytic pendulum ---------------------------------------------------------------------------------------------------------------

def test_pendulum_environments_saturate_at_their_own_limits(capi):
    """eight EFFORT_PENDULUM environments (I = 0.6 about the axis, URDF limit 1.5 N m, no gravity) in one batch, each with its own
    gains and limit: after one step v = e / I dt where the PD law asks for more than the environment's limit e, the implicit PD value
    elsewhere; in FORCE_AND_TORQUE the feed-forward torque is clipped to each environment's own limit"""
    from test_oracle_kat import EFFORT_PENDULUM
    I = 0.1 + 2.0 * 0.5 ** 2
    inf = np.inf
    #                 kp      kd    effort  target
    cases = np.array([[4000.0, 0.0, 1.5, 1.0],        # saturates at 1.5
                      [4000.0, 10.0, 3.0, -1.0],      # saturates at -3
                      [100.0, 2.0, 5.0, 0.01],        # 1 N m asked, 5 available: implicit PD with its own kd
                      [-1.0, -1.0, 0.5, 0.0002],      # batch gains (4000, 0): 0.8 N m asked, 0.5 available
                      [0.0, 0.0, -1.0, 1.0],          # no PD law
                      [50.0, 0.0, inf, 2.0],          # 100 N m asked, no limit
                      [4000.0, 0.0, 0.0, 1.0],        # an actuator that gives no torque
                      [-1.0, -1.0, -1.0, 0.0002]])    # all batch values: 0.8 N m asked, 1.5 available
    n = len(cases)
    bt = capi.Batch(capi.Model(EFFORT_PENDULUM), n)
    bt.set_params(gravity=(0.0, 0.0, 0.0))
    bt.set_control_mode(capi.PD_PLUS_FEEDFORWARD_TORQUE)
    bt.set_pd_gains(np.array([4000.0]), np.array([0.0]))
    bt.set_actuator_params(cases[:, None, :3].astype(np.float32))
    bt.set_state(np.zeros((n, 1), np.float32), np.zeros((n, 1), np.float32))
    bt.set_pd_target(cases[:, 3:4].astype(np.float32), np.zeros((n, 1), np.float32))
    bt.integrate(1)
    _, v = bt.get_state()
    kp = np.where(cases[:, 0] >= 0, cases[:, 0], 4000.0); kd = np.where(cases[:, 1] >= 0, cases[:, 1], 0.0)
    e = np.where(cases[:, 2] >= 0, cases[:, 2], 1.5)
    te = kp * cases[:, 3]
    soft = DT * kd + DT ** 2 * kp
    sat = np.abs(te) > e * (1 + soft / I)
    assert list(sat) == [True, True, False, True, False, False, True, False]
    expect = np.where(sat, np.sign(te) * e / I * DT, DT * te / (I + soft))
    assert np.allclose(v[:, 0], expect, rtol=2e-6, atol=1e-9), (v[:, 0], expect)
    # feed-forward alone, each environment's own limit
    bt.set_control_mode(capi.FORCE_AND_TORQUE)
    bt.set_state(np.zeros((n, 1), np.float32), np.zeros((n, 1), np.float32))
    tau = np.array([7.0, -7.0, 1.0, 0.2, 3.0, 100.0, 5.0, -2.0])
    bt.set_generalized_force(tau[:, None].astype(np.float32))
    bt.integrate(1)
    _, v = bt.get_state()
    clipped = np.clip(tau, -e, e)
    assert list(clipped) == [1.5, -3.0, 1.0, 0.2, 1.5, 100.0, 0.0, -1.5]
    assert np.allclose(v[:, 0], clipped / I * DT, rtol=2e-6, atol=1e-9), (v[:, 0], clipped / I * DT)
    assert np.allclose(bt.generalized_force()[:, 0], clipped, rtol=1e-6, atol=0)


# ---- 4: batch-level resolution and persistence ------------------------------------------------------------------------------------------

def test_minus_one_entries_follow_a_later_set_pd_gains(capi, monkeypatch):
    """rows of -1, then set_pd_gains, equal set_pd_gains alone; random rows with entries of -1, then set_pd_gains, equal the same rows
    with those entries resolved by hand to the new gains -- bit for bit"""
    n = 256
    out = {}
    for mode in ("all_minus_one", "never", "mixed", "resolved"):
        c = _setup(capi, monkeypatch, "quadruped_hm", n, seed=85)
        bt, t = c["bt"], c["t"]
        kp2, kd2 = 1.7 * c["kp"], 0.6 * c["kd"]
        rows = _random_rows(t, n, 19)
        if mode == "all_minus_one":
            bt.set_actuator_params(np.full((n, t["nv"], 3), -1.0, np.float32))
        elif mode == "mixed":
            bt.set_actuator_params(rows)
        bt.set_pd_gains(kp2, kd2)
        if mode == "resolved":
            r = rows.copy()
            r[:, :, 0] = np.where(r[:, :, 0] >= 0, r[:, :, 0], kp2.astype(np.float32))
            r[:, :, 1] = np.where(r[:, :, 1] >= 0, r[:, :, 1], kd2.astype(np.float32))
            bt.set_actuator_params(r)
        for k in range(4):
            bt.integrate(SUB)
        out[mode] = _outputs(bt)
    _same(out["never"], out["all_minus_one"], "rows of -1 after set_pd_gains: ")
    _same(out["resolved"], out["mixed"], "entries of -1 after set_pd_gains: ")
    assert out["never"]["gc"].tobytes() != out["mixed"]["gc"].tobytes()


def test_a_range_leaves_every_other_environment_alone(capi, monkeypatch):
    n, lo, hi = 300, 100, 200
    out = {}
    for mode in ("never", "range"):
        c = _setup(capi, monkeypatch, "quadruped_hm", n, seed=87)
        if mode == "range":
            c["bt"].set_actuator_params(_random_rows(c["t"], hi - lo, 21), env_begin=lo)
        for k in range(5):
            c["bt"].integrate(SUB)
        out[mode] = _outputs(c["bt"])
    keep = np.r_[0:lo, hi:n]
    for k in out["never"]:
        a, b = np.asarray(out["never"][k]), np.asarray(out["range"][k])
        assert a[keep].tobytes() == b[keep].tobytes(), f"{k} differs outside the range"
    assert (out["never"]["gc"][lo:hi] != out["range"]["gc"][lo:hi]).any(1).mean() > 0.9


def test_rows_survive_every_call_that_rebuilds_the_blob(capi, monkeypatch):
    """rows set before set_collision_friction, set_self_collision, set_heightmap, clear_terrain and set_params equal rows set after
    them, bit for bit, and differ from no rows"""
    n = 256
    out = {}
    for mode in ("before", "after", "none"):
        c = _setup(capi, monkeypatch, "generic_self", n, seed=89)
        bt, t = c["bt"], c["t"]
        rows = _random_rows(t, n, 23)
        if mode == "before":
            bt.set_actuator_params(rows)
        bt.set_collision_friction(1, 0.9)
        bt.set_self_collision(anymal_leg_pairs()[:6])
        H = (0.1 * np.random.default_rng(89).uniform(-1, 1, (49, 65))).astype(np.float32)
        bt.clear_terrain()
        bt.set_heightmap(65, 49, 12.8, 9.6, 0.1, -0.2, H)
        bt.set_params(mu=0.6)
        if mode == "after":
            bt.set_actuator_params(rows)
        for k in range(4):
            bt.integrate(SUB)
        out[mode] = _outputs(bt)
    _same(out["after"], out["before"], "rows set before the rebuilds: ")
    assert out["after"]["gc"].tobytes() != out["none"]["gc"].tobytes()


def test_gym_resets_keep_the_rows(capi, monkeypatch):
    """the gym task's steps and resets leave the rows in place: from the state they leave, the batch steps as a fresh batch with the
    same rows does, and unlike one without them"""
    n = 256
    g = _setup(capi, monkeypatch, "quadruped_hm", n, seed=91)
    rows = _random_rows(g["t"], n, 25)
    g["bt"].set_actuator_params(rows)
    gc_init = ANYMAL_GC0.copy(); gc_init[2] = 0.62
    g["bt"].gym_configure(gc_init, np.zeros(18), gc_init[7:], 0.6 * np.ones(12), [3, 6, 9, 12])
    g["bt"].gym_reset()
    rng = np.random.default_rng(5)
    obs = np.empty((n, 34), np.float32); rew = np.empty(n, np.float32); done = np.empty(n, np.uint8)
    base, terminated = rng.normal(0, 1.5, (n, 12)), 0
    for k in range(40):
        g["bt"].gym_step((base + rng.normal(0, 0.3, (n, 12))).astype(np.float32), SUB, obs, rew, done)
        terminated += int(done.sum())
    assert terminated > 10
    gc, gv = g["bt"].get_state()
    res = {}
    for mode, b in (("gym", g["bt"]), ("same", None), ("none", None)):
        if b is None:
            b = _setup(capi, monkeypatch, "quadruped_hm", n, seed=91)["bt"]
            if mode == "same":
                b.set_actuator_params(rows)
        b.set_state(gc, gv); b.set_pd_target(gc, np.zeros((n, 18), np.float32))
        for k in range(3):
            b.integrate(SUB)
        res[mode] = b.get_state()[0]
    assert res["gym"].tobytes() == res["same"].tobytes()
    assert res["gym"].tobytes() != res["none"].tobytes()


# ---- 5: the gym task on rows alone ------------------------------------------------------------------------------------------------------

def _quat_rot(q):
    w, x, y, z = q
    return np.array([[1 - 2 * (y * y + z * z), 2 * (x * y - w * z), 2 * (x * z + w * y)],
                     [2 * (x * y + w * z), 1 - 2 * (x * x + z * z), 2 * (y * z - w * x)],
                     [2 * (x * z - w * y), 2 * (y * z + w * x), 1 - 2 * (x * x + y * y)]])


def test_gym_step_runs_on_rows_without_set_pd_gains(capi):
    """gym_step with per-environment gains and no set_pd_gains: one launch per control step, and states, observations and rewards
    equal those of control_step with the same targets and rows (the targets action * std + mean, std a power of two so that the
    product is exact whether or not it is fused)"""
    n = 256
    path = os.path.join(RSC, "anymal_c_like.urdf")
    rng = np.random.default_rng(93)
    rows = np.full((n, 18, 3), -1.0, np.float32)
    rows[:, 6:, 0] = rng.uniform(80.0, 200.0, (n, 12)); rows[:, 6:, 1] = rng.uniform(1.0, 4.0, (n, 12))
    rows[:, 6:, 2] = rng.uniform(30.0, 80.0, (n, 12))
    gc_init = ANYMAL_GC0.copy(); gc_init[2] = 0.57
    std = 0.5 * np.ones(12)
    bts = {}
    for mode in ("gym", "ref"):
        bt = capi.Batch(capi.Model(path), n)
        bt.set_ground(0.0)
        bt.set_params(threshold=THRESH)
        bt.set_control_mode(capi.PD_PLUS_FEEDFORWARD_TORQUE)
        bt.set_actuator_params(rows)
        bts[mode] = bt
    g, r = bts["gym"], bts["ref"]
    plain = capi.Batch(capi.Model(path), 4)            # neither gains nor rows: refused
    plain.gym_configure(gc_init, np.zeros(18), gc_init[7:], std, [3, 6, 9, 12])
    plain.gym_reset()
    assert capi.lib().rsb_batch_gym_step(plain.h, np.zeros((4, 12), np.float32).ctypes.data_as(C.c_void_p), capi.HOST, SUB, None, None, None, capi.HOST) == -1
    assert b"rsb_batch_set_actuator_params" in capi.lib().rsb_last_error()
    g.gym_configure(gc_init, np.zeros(18), gc_init[7:], std, [3, 6, 9, 12])
    g.gym_reset()
    gc0 = np.tile(gc_init, (n, 1)).astype(np.float32)
    r.set_state(gc0, np.zeros((n, 18), np.float32))
    obs = np.empty((n, 34), np.float32); rew = np.empty(n, np.float32); done = np.empty(n, np.uint8)
    robs = np.empty((n, 34), np.float32)
    alive = np.ones(n, bool)
    L0 = g.launch_count()
    for k in range(6):
        act = rng.normal(0, 0.4, (n, 12)).astype(np.float32)
        g.gym_step(act, SUB, obs, rew, done)
        pt = gc0.copy(); pt[:, 7:] = act * std.astype(np.float32) + gc_init[7:].astype(np.float32)
        r.control_step(pt, SUB, robs, vtarget=np.zeros((n, 18), np.float32))
        alive &= done == 0
        gg, gv = g.get_state(); rg, rv = r.get_state()
        assert gg[alive].tobytes() == rg[alive].tobytes() and gv[alive].tobytes() == rv[alive].tobytes(), f"control step {k}"
        assert obs[alive].tobytes() == robs[alive].tobytes()
        tau = r.generalized_force().astype(np.float64)
        vbx = np.array([(_quat_rot(rg[e, 3:7].astype(np.float64)).T @ rv[e, :3])[0] for e in range(n)])
        ref = -4e-5 * (tau ** 2).sum(1) + 0.3 * np.minimum(4.0, vbx)
        assert np.abs(rew - ref)[alive].max() < 1e-5 * (1 + np.abs(ref).max())
    assert g.launch_count() == L0 + 6
    assert alive.mean() > 0.9


# ---- 6: launch shapes and sources ------------------------------------------------------------------------------------------------------

@pytest.mark.parametrize("which", list(SETUPS))
def test_every_launch_shape_gives_the_same_results(capi, monkeypatch, which):
    """a distinct row in every environment: every CTA size that fits, the sub-step barrier and the paired stage A on and off, a
    partly filled last round -- the same results bit for bit"""
    n = 2300 if which.startswith("humanoid") else 4500
    ref, taken = None, []
    shapes = [(None, "1", "1")] + [(w, "1", "1") for w in (28, 16, 14, 8, 4, 1)] + [(None, "0", "1"), (None, "1", "0")]
    for wpc, barrier, pair in shapes:
        monkeypatch.setenv("RSB_SUBSTEP_BARRIER", barrier); monkeypatch.setenv("RSB_PAIR_STAGE_A", pair)
        c = _setup(capi, monkeypatch, which, n, seed=95, wpc=wpc)
        if wpc is not None and c["cfg"]["wpc"] != wpc:
            continue                                                          # did not fit
        taken.append(c["cfg"]["wpc"])
        c["bt"].set_actuator_params(_random_rows(c["t"], n, 27))
        for k in range(2):
            c["bt"].integrate(SUB)
        o = _outputs(c["bt"])
        res = tuple(np.asarray(v).tobytes() for v in o.values())
        if ref is None:
            ref = res
            T = c["cfg"]["wpc"] * c["cfg"]["grid"]
            assert n % T != 0 and o["cnt"].any()
        assert res == ref, f"{which}: differs at wpc {wpc} barrier {barrier} pairing {pair}"
        del c
    assert len(set(taken)) >= 3


def test_pinned_pageable_device_and_pybind_sources_agree(capi, monkeypatch):
    import torch
    from raisimlib_b200 import _rsb_py
    n = 200
    out = {}
    for mode in ("pageable", "pinned", "device", "raw"):
        c = _setup(capi, monkeypatch, "quadruped_hm", n, seed=97)
        bt = c["bt"]
        rows = _random_rows(c["t"], n, 29)
        if mode == "pageable":
            bt.set_actuator_params(rows[50:], env_begin=50); bt.set_actuator_params(rows[:50])
        elif mode == "pinned":
            p = torch.from_numpy(rows).pin_memory()
            assert capi.lib().rsb_batch_set_actuator_params(bt.h, C.c_void_p(p.data_ptr()), 0, n, capi.HOST) == 0
        elif mode == "device":
            bt.set_actuator_params_from(torch.from_numpy(rows).cuda())
        elif mode == "raw":
            tr = torch.from_numpy(rows).cuda()
            assert capi.lib().rsb_batch_set_actuator_params(bt.h, C.c_void_p(tr.data_ptr()), 0, n, capi.DEVICE) == 0
        for k in range(3):
            bt.integrate(SUB)
        out[mode] = _outputs(bt)
    for mode in ("pinned", "device", "raw"):
        _same(out["pageable"], out[mode], f"{mode} source: ")
    c = _setup(capi, monkeypatch, "quadruped_hm", n, seed=97)
    with pytest.raises(ValueError):
        c["bt"].set_actuator_params_from(torch.from_numpy(rows).double().cuda())
    with pytest.raises(ValueError):
        c["bt"].set_actuator_params_from(torch.from_numpy(rows[:, :-1].copy()).cuda())
    with pytest.raises(ValueError):
        c["bt"].set_actuator_params_from(torch.from_numpy(np.ascontiguousarray(rows.transpose(1, 0, 2))).cuda().transpose(0, 1))
    with pytest.raises(ValueError):
        c["bt"].set_actuator_params_from(torch.from_numpy(rows))
    with pytest.raises(ValueError):
        c["bt"].set_actuator_params(rows[:, :, :2])
    # the pybind module against the ctypes binding: same rows from the device, same state through DLPack
    monkeypatch.delenv("RSB_FORCE_WPC", raising=False); monkeypatch.setenv("RSB_FORCE_GENERIC", "0")
    path = os.path.join(RSC, "anymal_c_like.urdf")
    pb = _rsb_py.Batch(_rsb_py.Model(path), n, 0)
    bt = capi.Batch(capi.Model(path), n)
    gc = c["gc"]
    pb.set_ground(0.0); bt.set_ground(0.0)
    torch.from_dlpack(pb.gc()).copy_(torch.from_numpy(gc).cuda())
    torch.from_dlpack(pb.gv()).copy_(torch.from_numpy(c["gv"]).cuda())
    bt.set_state(gc, c["gv"])
    torch.from_dlpack(pb.pd_target()).copy_(torch.from_numpy(gc).cuda())      # both in PD mode without set_pd_gains: the rows' gains alone
    bt.set_pd_target(gc, np.zeros((n, 18), np.float32))
    tr = torch.from_numpy(rows).cuda()
    torch.cuda.synchronize()
    pb.set_actuator_params(tr.data_ptr(), 0, n); bt.set_actuator_params(rows)
    pb.integrate(SUB); bt.integrate(SUB); pb.sync()
    assert torch.from_dlpack(pb.gc()).cpu().numpy().tobytes() == bt.get_state()[0].tobytes()


# ---- 7: refusals and launches ------------------------------------------------------------------------------------------------------

def test_refusals_change_nothing(capi, monkeypatch):
    import torch
    n = 200
    L = capi.lib()
    assert L.rsb_batch_set_actuator_params(None, None, 0, 1, capi.HOST) == -1
    assert L.rsb_batch_clear_actuator_params(None) == -1
    runs = {}
    for mode in ("clean", "refused", "first_refused", "never"):
        c = _setup(capi, monkeypatch, "quadruped_hm", n, seed=99)
        bt, nv = c["bt"], c["t"]["nv"]
        rows = _random_rows(c["t"], n, 31)
        if mode == "clean":
            bt.set_actuator_params(rows)
        if mode in ("refused", "first_refused"):
            if mode == "refused":
                bt.set_actuator_params(rows)
            L0 = bt.launch_count()
            bad = [(np.nan, f) for f in range(3)] + [(np.inf, 0), (-np.inf, 0), (np.inf, 1), (-np.inf, 1), (-np.inf, 2)]
            names = ("kp", "kd", "effort limit")
            for v, f in bad:
                for e, i in ((0, 0), (57, nv // 2), (n - 1, nv - 1)):
                    r = rows.copy(); r[e, i, f] = v
                    for where in (capi.HOST, capi.DEVICE):
                        src = torch.from_numpy(r).cuda() if where == capi.DEVICE else r
                        ptr = C.c_void_p(src.data_ptr()) if where == capi.DEVICE else r.ctypes.data_as(C.c_void_p)
                        assert L.rsb_batch_set_actuator_params(bt.h, ptr, 0, n, where) == -1, (v, f, e, i)
                        assert b"no row changed" in L.rsb_last_error()
                        assert f"environment {e}, dof {i}: {names[f]}".encode() in L.rsb_last_error(), L.rsb_last_error()
            ok = rows.ctypes.data_as(C.c_void_p)
            for begin, count, where in ((n - 1, 2, capi.HOST), (-1, 1, capi.HOST), (0, -1, capi.HOST), (0, n, 2), (0, n, -1)):
                assert L.rsb_batch_set_actuator_params(bt.h, ok, begin, count, where) == -1, (begin, count, where)
            assert L.rsb_batch_set_actuator_params(bt.h, None, 0, n + 1, capi.HOST) == -1
            assert bt.launch_count() == L0
        runs[mode] = []
        for k in range(3):
            bt.integrate(SUB)
            runs[mode].append(_outputs(bt))
    for k in range(3):
        _same(runs["clean"][k], runs["refused"][k], f"after refusals, step {k}: ")
        _same(runs["never"][k], runs["first_refused"][k], f"refused first call, step {k}: ")


def test_rows_add_no_launch(capi, monkeypatch):
    """setting, resetting and clearing rows launches nothing the batch counts, leaves the getters' buffers fresh, and a step with rows is
    one launch"""
    n = 128
    c = _setup(capi, monkeypatch, "quadruped_hm", n, seed=101)
    bt = c["bt"]
    bt.mass_matrix()
    L0 = bt.launch_count()
    bt.set_actuator_params(_random_rows(c["t"], n, 33))
    bt.set_actuator_params(None, env_begin=10, env_count=5)
    bt.mass_matrix()
    assert bt.launch_count() == L0
    bt.integrate(SUB)
    assert bt.launch_count() == L0 + 1
    bt.clear_actuator_params()
    bt.integrate(SUB)
    assert bt.launch_count() == L0 + 2


# ---- 8: the C++ facade ------------------------------------------------------------------------------------------------------------------

def test_cpp_gain_randomization_example():
    """the raisim:: facade: setPdGains and setActuationLimits in an upstream-shaped reset(), one launch per control step, every
    environment equal to a stand-alone World with the same gains and limits (examples/gain_randomization.cpp)"""
    exe = os.path.join(ROOT, "examples", "gain_randomization")
    if not os.path.exists(exe):
        subprocess.check_call(["make", "-C", os.path.join(ROOT, "examples")])
    out = subprocess.run([exe, os.path.join(RSC, "anymal_c_like.urdf")], capture_output=True, text=True, timeout=600)
    print(out.stdout)
    assert out.returncode == 0, out.stdout + out.stderr
