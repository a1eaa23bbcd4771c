"""IMU readings over a whole launch (rsb_batch_set_imus / rsb_batch_get_imu_readings), through the C-ABI on an H100 (pytest -m gpu):
the step kernel's readings against the float64 restatement tests/imu_ref.py on the GPU's own trajectory, with every per-environment
feature on, known answers, no effect on the physics, the launch rules (shapes, which launches write, gym terminations, launch count,
batch size), refusals, the pybind module and the C++ facade."""
import ctypes as C
import os
import subprocess

import numpy as np
import pytest

from conftest import ROOT, RSC
from frame_ref import random_frames
from helpers import ANYMAL_GC0, PENDULUM_URDF, quat_to_rot
from imu_ref import imu_substep
from oracle.urdf_tables import load_tables
from test_gpu_contact_forces import _make, _outputs, _same
from test_gpu_feature_mix import _batch as _mix_batch, _command as _mix_command, _inputs as _mix_inputs, _wrench as _mix_wrench
from test_self_collision_oracle import anymal_leg_pairs

pytestmark = pytest.mark.gpu

SUB, DT = 4, 0.0025
REL_F, ABS_F, REL_W, ABS_W = 1e-3, 2e-2, 1e-3, 1e-4
ROT = quat_to_rot(np.array([0.9, 0.2, -0.3, 0.25]) / np.linalg.norm([0.9, 0.2, -0.3, 0.25])).astype(np.float32)
SPIN_URDF = """<robot name="spin">
  <link name="world"/>
  <link name="arm"><inertial><origin xyz="0.3 0.1 0"/><mass value="1.0"/><inertia ixx="0.01" ixy="0" ixz="0" iyy="0.02" iyz="0" izz="0.03"/></inertial></link>
  <joint name="j" type="revolute"><parent link="world"/><child link="arm"/><origin xyz="0 0 0.5"/><axis xyz="0 0 1"/></joint>
</robot>"""


@pytest.fixture(scope="module")
def capi():
    import torch
    assert torch.cuda.is_available(), "GPU tests need a CUDA device"
    from raisimlib_b200 import capi as c
    return c


def _sensors(t, rng, feet=True):
    """the base at its origin, the feet (ANYmal-like model) or random bodies, and a rotated frame off a random body's origin"""
    nb = t["nb"]
    body = [0] + ([3, 6, 9, 12] if feet and nb == 13 else list(rng.integers(1, nb, 4)))
    pos = np.zeros((len(body), 3), np.float32)
    pos[1:] = rng.uniform(-0.1, 0.1, (len(body) - 1, 3))
    rot = np.tile(np.eye(3, dtype=np.float32), (len(body), 1, 1))
    rb, rp, rr = random_frames(rng, nb, 2)
    return np.r_[body, rb].astype(np.int32), np.r_[pos, rp], np.r_[rot, rr]


def _check(got, ref, rel, ab, what):
    err = np.abs(got.astype(np.float64) - ref)
    lim = rel * np.linalg.norm(ref, axis=-1, keepdims=True) + ab
    bad = ~(err <= lim)
    assert not bad.any(), f"{what}: {bad.sum()} entries off, worst {err.max():.3e} (limit there {lim.reshape(-1)[np.argmax(err)]:.3e})"


def _against_reference(capi, a, b, t, sensors, steps, before=None, command=None):
    """a steps one launch of SUB sub-steps per control step, b the same sub-steps as launches of one; states equal bit for bit; b's
    readings of every sub-step and a's of the launch against imu_ref on b's trajectory"""
    body, pos, rot = sensors
    g = np.array(a.get_params().gravity[:], np.float64)
    for bt in (a, b):
        bt.set_imus(body, pos, rot)
    for k in range(steps):
        for bt in (a, b):
            if command:
                command(bt, k)
        if before:
            before(a, k)
        a.integrate(SUB)
        gc, gv = b.get_state()
        fs, ws = [], []
        for s in range(SUB):
            if before:
                before(b, k)
            b.integrate(1)
            gc1, gv1 = b.get_state()
            ref = [imu_substep(t, gc[e], gv[e], gv1[e], DT, body, pos, rot, g) for e in range(len(gc))]
            f_ref, w_ref = np.stack([r[0] for r in ref]), np.stack([r[1] for r in ref])
            f1, w1 = b.imu_readings()
            _check(f1, f_ref, REL_F, ABS_F, f"step {k} sub-step {s} specific force")
            _check(w1, w_ref, REL_W, ABS_W, f"step {k} sub-step {s} angular rate")
            fs.append(f_ref); ws.append(w_ref)
            gc, gv = gc1, gv1
        assert a.get_state()[0].tobytes() == b.get_state()[0].tobytes() and a.get_state()[1].tobytes() == b.get_state()[1].tobytes()
        lin, ang = a.imu_readings()
        _check(lin, np.mean(fs, 0), REL_F, ABS_F, f"step {k} launch specific force")
        _check(ang, np.mean(ws, 0), REL_W, ABS_W, f"step {k} launch angular rate")
        assert not a.diverged().any()
    return lin


# ---- 1: against the reference on the GPU's own trajectory -------------------------------------------------------------------------

@pytest.mark.parametrize("case", ["quadruped_hm_paired", "quadruped_hm_unpaired", "humanoid", "generic_self", "quadruped_DL", "quadruped_AN"])
def test_readings_match_the_reference(capi, monkeypatch, case):
    """64 environments, 3 control steps: the quadruped instance on a height map with paired stage A on and off, the humanoid on the
    ground, the generic instance with self-collision pairs, the actuation-delay (DL) and actuator-network (AN) instances"""
    name = case.split("_")[0]
    monkeypatch.setenv("RSB_PAIR_STAGE_A", "0" if case.endswith("unpaired") else "1")
    terrain = "hm" if case.startswith("quadruped_hm") else "ground"
    n, seed = 64, 500 + len(case)
    a, b = (_make(capi, monkeypatch, name, n, terrain, seed=seed, oracles=False) for _ in range(2))
    for c in (a, b):
        if case == "generic_self":
            c["bt"].set_self_collision(anymal_leg_pairs())
        if case == "quadruped_DL":
            c["bt"].set_actuation_delay((np.arange(n) % 5).astype(np.int32))
        if case == "quadruped_AN":
            rng = np.random.default_rng(3)
            layers = [(rng.uniform(-0.5, 0.5, (16, 6)).astype(np.float32), rng.uniform(-0.1, 0.1, 16).astype(np.float32)),
                      (rng.uniform(-2, 2, (1, 16)).astype(np.float32), np.zeros(1, np.float32))]
            c["bt"].set_actuator_network(list(range(6, 18)), layers, 3)
        c["bt"].set_state(c["gc"], c["gv"])
    sensors = _sensors(a["t"], np.random.default_rng(seed))
    lin = _against_reference(capi, a["bt"], b["bt"], a["t"], sensors, 3)
    assert np.abs(lin).max() > 1.0


@pytest.mark.parametrize("name", ["anymal", "atlas"])
def test_every_feature_at_once_matches_the_reference(capi, monkeypatch, name):
    """inertia, friction and actuator rows, an actuator network, actuation delays, an external wrench in the first control step (on
    every launch of it: a wrench lasts one launch), contact bodies, frames and a height scan all set"""
    x = _mix_inputs(name, "AN+DL", 32, seed=41)
    a, b = _mix_batch(capi, monkeypatch, x), _mix_batch(capi, monkeypatch, x)
    sensors = _sensors(x["t"], np.random.default_rng(42))
    _against_reference(capi, a, b, x["t"], sensors, 3, before=lambda bt, k: _mix_wrench(bt, x) if k == 0 else None,
                       command=lambda bt, k: _mix_command(bt, x, k))


# ---- 2: known answers ---------------------------------------------------------------------------------------------------------------

def test_known_answers(capi, monkeypatch):
    monkeypatch.delenv("RSB_FORCE_WPC", raising=False); monkeypatch.setenv("RSB_FORCE_GENERIC", "0")
    # the welded root of a fixed-base robot is at rest: -g in the sensor frame, exactly 0 rate
    bt = capi.Batch(capi.Model(PENDULUM_URDF), 16)
    bt.set_state(np.random.default_rng(1).uniform(-1, 1, (16, 3)).astype(np.float32), np.zeros((16, 3), np.float32))
    bt.set_imus([0], np.array([[0.1, 0.2, 0.3]], np.float32), ROT[None])
    bt.integrate(SUB)
    lin, ang = bt.imu_readings()
    assert np.abs(lin - ROT.T @ np.array([0, 0, 9.81], np.float32)).max() < 1e-5 and not ang.any()
    # free fall: a quadruped at rest with no terrain and no torques reads 0 on every body, launch after launch
    c = _make(capi, monkeypatch, "quadruped", 64, "ground", seed=7, oracles=False)
    bt = c["bt"]
    bt.clear_terrain(); bt.set_control_mode(capi.FORCE_AND_TORQUE)
    gc = c["gc"].copy(); gc[:, 2] = 5.0
    bt.set_state(gc, np.zeros_like(c["gv"]))
    bt.set_imus(*_sensors(c["t"], np.random.default_rng(8)))
    for _ in range(5):
        bt.integrate(SUB)
        lin, ang = bt.imu_readings()
        assert np.abs(lin).max() < 1e-3 and np.abs(ang).max() < 1e-5
    # standing still on the ground: the base reads +|g| opposite to gravity in its own frame
    c = _make(capi, monkeypatch, "quadruped", 64, "ground", seed=9, oracles=False)
    bt = c["bt"]
    gc = np.tile(ANYMAL_GC0.astype(np.float32), (64, 1)); gc[:, :2] = c["gc"][:, :2]; gc[:, 2] = 0.56
    bt.set_pd_target(gc, np.zeros((64, 18), np.float32))
    bt.set_state(gc, np.zeros((64, 18), np.float32))
    bt.set_imus([0], np.zeros((1, 3), np.float32))
    for _ in range(150):
        bt.integrate(SUB)
    lin, ang = bt.imu_readings()
    q = bt.get_state()[0][:, 3:7].astype(np.float64)
    up = np.stack([quat_to_rot(x).T @ np.array([0, 0, 9.81]) for x in q])
    assert np.abs(lin - up).max() < 0.05 and np.abs(ang).max() < 0.01
    # a link spinning at a constant rate in zero gravity: the centripetal -w^2 r_perp and the rate w
    bt = capi.Batch(capi.Model(SPIN_URDF), 8)
    bt.set_params(gravity=(0.0, 0.0, 0.0))
    w = np.linspace(-6, 6, 8).astype(np.float32)
    bt.set_state(np.zeros((8, 1), np.float32), w[:, None])
    pos = np.array([[0.4, -0.2, 0.1]], np.float32)
    bt.set_imus([1], pos, ROT[None])
    for _ in range(3):
        bt.integrate(SUB)
    lin, ang = bt.imu_readings()
    q, v = bt.get_state()
    assert np.abs(v[:, 0] - w).max() < 1e-4
    for e in range(8):
        # the sensor frame turns with the link: the centripetal acceleration is -w^2 (x, y, 0) in the link frame whatever the angle;
        # over a launch the reading averages sub-step readings in the same link-fixed frame
        f_link = -float(w[e]) ** 2 * np.array([pos[0, 0], pos[0, 1], 0.0])
        assert np.abs(lin[e] - ROT.T @ f_link).max() < 1e-3 * (1 + abs(w[e]) ** 2)
        assert np.abs(ang[e] - ROT.T @ np.array([0, 0, w[e]])).max() < 1e-5


# ---- 3: no effect on the physics ------------------------------------------------------------------------------------------------

@pytest.mark.parametrize("case", ["quadruped", "humanoid", "generic", "quadruped_DL", "quadruped_AN"])
def test_sensors_change_nothing_else(capi, monkeypatch, case):
    name = case.split("_")[0]
    runs = []
    for with_imus in (False, True):
        c = _make(capi, monkeypatch, name, 256, "hm" if name == "quadruped" else "ground", seed=31, oracles=False)
        bt = c["bt"]
        if name == "generic":
            bt.set_self_collision(anymal_leg_pairs())
        if case == "quadruped_DL":
            bt.set_actuation_delay((np.arange(256) % 7).astype(np.int32))
        if case == "quadruped_AN":
            rng = np.random.default_rng(4)
            bt.set_actuator_network(list(range(6, 18)), [(rng.uniform(-0.5, 0.5, (8, 6)).astype(np.float32), np.zeros(8, np.float32)),
                                                         (rng.uniform(-1, 1, (1, 8)).astype(np.float32), np.zeros(1, np.float32))], 3)
        bt.set_contact_bodies(list(range(min(32, c["t"]["nb"]))))
        if with_imus:
            bt.set_imus(*_sensors(c["t"], np.random.default_rng(5)))
        bt.set_state(c["gc"], c["gv"])
        for _ in range(3):
            bt.integrate(SUB)
        o = _outputs(bt)
        o["f"], o["s"] = bt.body_contact_forces()
        runs.append(o)
    _same(runs[0], runs[1], f"{case}: ")


# ---- 4: launch behaviour ------------------------------------------------------------------------------------------------------------

def test_every_launch_shape_gives_the_same_readings(capi, monkeypatch):
    """every CTA size that fits, the sub-step barrier and the paired stage A on and off; the batch ends on a partly filled round"""
    n, ref, taken = 4500, None, []
    shapes = [(None, "1", "1")] + [(w, "1", "1") for w in (28, 16, 14, 8, 4, 1)] + [(None, "0", "1"), (None, "1", "0")]
    for wpc, barrier, pair in shapes:
        monkeypatch.setenv("RSB_SUBSTEP_BARRIER", barrier); monkeypatch.setenv("RSB_PAIR_STAGE_A", pair)
        c = _make(capi, monkeypatch, "quadruped", n, "hm", seed=61, wpc=wpc, oracles=False)
        if wpc is not None and c["cfg"]["wpc"] != wpc:
            continue                                                          # did not fit
        taken.append(c["cfg"]["wpc"])
        c["bt"].set_imus(*_sensors(c["t"], np.random.default_rng(6)))
        for _ in range(2):
            c["bt"].integrate(SUB)
        r = c["bt"].imu_readings()
        if ref is None:
            ref = r
        assert r[0].tobytes() == ref[0].tobytes() and r[1].tobytes() == ref[1].tobytes(), f"differs at wpc {wpc} barrier {barrier} pairing {pair}"
        del c
    assert len(set(taken)) >= 5


def test_which_launches_write(capi, monkeypatch):
    import torch
    c = _make(capi, monkeypatch, "quadruped", 128, "hm", seed=11, oracles=False)
    bt = c["bt"]
    sensors = _sensors(c["t"], np.random.default_rng(12))
    bt.set_imus(*sensors)
    lin, ang = bt.imu_readings()
    assert lin.shape == (128, len(sensors[0]), 3) and not lin.any() and not ang.any()          # zero until an advancing launch
    launches = bt.launch_count()
    bt.integrate(SUB)
    assert bt.launch_count() == launches + 1                                                     # no extra launch
    ref = bt.imu_readings()
    assert np.abs(ref[0]).max() > 1.0
    tl, ta = torch.zeros((128, len(sensors[0]), 3), device="cuda"), torch.zeros((128, len(sensors[0]), 3), device="cuda")
    launches = bt.launch_count()
    bt.imu_readings_into(tl, ta); bt.sync()
    assert bt.launch_count() == launches and tl.cpu().numpy().tobytes() == ref[0].tobytes() and ta.cpu().numpy().tobytes() == ref[1].tobytes()
    sl = bt.imu_readings(37, 50)
    assert sl[0].tobytes() == ref[0][37:87].tobytes() and sl[1].tobytes() == ref[1][37:87].tobytes()
    with pytest.raises(ValueError):
        bt.imu_readings_into(torch.zeros((128, len(sensors[0]), 3), dtype=torch.float64, device="cuda"))
    # launches that do not advance the state leave them alone
    bt.set_frames([0, 3], np.zeros((2, 3), np.float32))
    bt.set_height_scan([0, 0], np.array([[0.1, 0.0], [0.0, 0.1]], np.float32))
    bt.integrate1(); bt.update_kinematics(); bt.frame_states(); bt.frame_jacobians(); bt.height_scan(); bt.mass_matrix()
    bt.set_state(c["gc"], c["gv"])                                  # a state write changes nothing until the next launch
    r = bt.imu_readings()
    assert r[0].tobytes() == ref[0].tobytes() and r[1].tobytes() == ref[1].tobytes()
    # integrate2 and control_step advance the state and write
    bt.integrate2()
    r2 = bt.imu_readings()
    assert r2[0].tobytes() != ref[0].tobytes()
    d = _make(capi, monkeypatch, "quadruped", 128, "hm", seed=11, oracles=False)
    d["bt"].set_imus(*sensors)
    pin_t = torch.from_numpy(d["pt"]).pin_memory()
    d["bt"].control_step(pin_t, SUB, None)
    r3 = d["bt"].imu_readings()
    assert r3[0].tobytes() == ref[0].tobytes() and r3[1].tobytes() == ref[1].tobytes()
    # a new list reads zero until the next step
    bt.set_imus_by_frame(["base", "LF_FOOT"])
    lin, ang = bt.imu_readings()
    assert lin.shape == (128, 2, 3) and not lin.any() and not ang.any()


def test_gym_termination_keeps_the_readings_of_the_step_that_ended_it(capi, monkeypatch):
    """the gym step's readings equal those of the same sub-steps as a plain integrate from the same state and targets, terminated
    environments included (action_std 1, action_mean 0: the targets are the actions themselves)"""
    n, feet = 128, [3, 6, 9, 12]
    g = _make(capi, monkeypatch, "quadruped", n, "ground", seed=72, oracles=False)
    p = _make(capi, monkeypatch, "quadruped", n, "ground", seed=72, oracles=False)
    sensors = _sensors(g["t"], np.random.default_rng(13))
    g["bt"].set_imus(*sensors); p["bt"].set_imus(*sensors)
    gc_init = g["gc"][0].copy(); gc_init[2] = 0.54; gc_init[3:7] = [1, 0, 0, 0]
    g["bt"].gym_configure(gc_init, np.zeros(18), np.zeros(12), np.ones(12), feet)
    g["bt"].gym_reset()
    rng = np.random.default_rng(5)
    obs = np.empty((n, 34), np.float32); rew = np.empty(n, np.float32); done = np.empty(n, np.uint8)
    base = gc_init[7:] + rng.normal(0, 1.5, (n, 12))
    terminated = 0
    for k in range(40):
        act = (base + rng.normal(0, 0.3, (n, 12))).astype(np.float32)
        gc, gv = g["bt"].get_state()
        pt = np.tile(gc_init.astype(np.float32), (n, 1)); pt[:, 7:] = act
        p["bt"].set_state(gc, gv); p["bt"].set_pd_target(pt, np.zeros((n, 18), np.float32))
        p["bt"].integrate(SUB)
        g["bt"].gym_step(act, SUB, obs, rew, done)
        rg, rp = g["bt"].imu_readings(), p["bt"].imu_readings()
        assert rg[0].tobytes() == rp[0].tobytes() and rg[1].tobytes() == rp[1].tobytes(), f"control step {k}"
        terminated += int(done.sum())
    assert terminated > 5


def test_a_batch_of_256_equals_batches_of_one(capi, monkeypatch):
    c = _make(capi, monkeypatch, "quadruped", 256, "hm", seed=21, oracles=False)
    sensors = _sensors(c["t"], np.random.default_rng(22))
    c["bt"].set_imus(*sensors)
    c["bt"].integrate(SUB); c["bt"].integrate(SUB)
    lin, ang = c["bt"].imu_readings()
    for e in (0, 101, 255):
        one = _make(capi, monkeypatch, "quadruped", 1, "hm", seed=21, oracles=False)
        one["bt"].set_pd_target(c["pt"][e:e + 1], np.zeros((1, 18), np.float32))
        one["bt"].set_state(c["gc"][e:e + 1], c["gv"][e:e + 1])
        one["bt"].set_imus(*sensors)
        one["bt"].integrate(SUB); one["bt"].integrate(SUB)
        l1, a1 = one["bt"].imu_readings()
        assert l1.tobytes() == lin[e:e + 1].tobytes() and a1.tobytes() == ang[e:e + 1].tobytes(), f"environment {e}"


# ---- 5: refusals ------------------------------------------------------------------------------------------------------------------------

def test_refusals_change_nothing(capi, monkeypatch):
    c = _make(capi, monkeypatch, "quadruped", 64, "ground", seed=51, oracles=False)
    bt, L = c["bt"], capi.lib()
    with pytest.raises(capi.RsbError, match="no IMUs"):
        bt.nimus = 1; bt.imu_readings()
    sensors = _sensors(c["t"], np.random.default_rng(52))
    bt.set_imus(*sensors)
    bt.integrate(SUB)
    ref = bt.imu_readings()
    P = lambda a, dt=np.float32: np.ascontiguousarray(a, dt).ctypes.data_as(C.c_void_p)
    good_b, good_p = [0, 3], np.zeros((2, 3))
    skew = np.tile(np.eye(3), (2, 1, 1)); skew[1, 0, 1] = 1e-3                       # |R^T R - I| = 1e-3
    mirror = np.tile(np.eye(3), (2, 1, 1)); mirror[1, 2, 2] = -1.0                   # det -1
    nan_p = good_p.copy(); nan_p[1, 1] = np.nan
    inf_r = np.tile(np.eye(3), (2, 1, 1)); inf_r[0, 0, 0] = np.inf
    calls = [(None, P(good_p), None, 2), (P(good_b, np.int32), None, None, 2), (P([0] * 9, np.int32), P(np.zeros((9, 3))), None, 9),
             (P(good_b, np.int32), P(good_p), None, -1), (P([0, 13], np.int32), P(good_p), None, 2), (P([-1, 0], np.int32), P(good_p), None, 2),
             (P(good_b, np.int32), P(nan_p), None, 2), (P(good_b, np.int32), P(good_p), P(inf_r), 2),
             (P(good_b, np.int32), P(good_p), P(skew), 2), (P(good_b, np.int32), P(good_p), P(mirror), 2)]
    for k, (b, p, r, cnt) in enumerate(calls):
        assert L.rsb_batch_set_imus(bt.h, b, p, r, cnt) == -1 and L.rsb_last_error(), f"call {k} was accepted"
    assert L.rsb_batch_set_imus(None, P(good_b, np.int32), P(good_p), None, 2) == -1
    out = np.zeros((64, len(sensors[0]), 3), np.float32)
    for begin, count, where in ((60, 5, 0), (-1, 2, 0), (0, 64, 7)):
        assert L.rsb_batch_get_imu_readings(bt.h, begin, count, P(out), None, where) == -1
    r = bt.imu_readings()
    assert r[0].tobytes() == ref[0].tobytes() and r[1].tobytes() == ref[1].tobytes()
    # a rotation within the tolerance is taken; the sensors set before the refusals are still the ones that step
    d = _make(capi, monkeypatch, "quadruped", 64, "ground", seed=51, oracles=False)
    d["bt"].set_imus(*sensors)
    for x in (bt, d["bt"]):
        x.set_state(c["gc"], c["gv"]); x.integrate(SUB)
    assert bt.imu_readings()[0].tobytes() == d["bt"].imu_readings()[0].tobytes()
    near = np.tile(np.eye(3), (2, 1, 1)); near[1, 0, 1] = 2e-5
    bt.set_imus(good_b, good_p, near)
    bt.set_imus([], np.zeros((0, 3)))
    with pytest.raises(capi.RsbError, match="no IMUs"):
        bt.nimus = 1; bt.imu_readings()


# ---- 6: the pybind module and the C++ facade --------------------------------------------------------------------------------------

def test_pybind_module_fills_torch_tensors(capi, monkeypatch):
    import torch
    from raisimlib_b200 import _rsb_py
    monkeypatch.delenv("RSB_FORCE_WPC", raising=False); monkeypatch.setenv("RSB_FORCE_GENERIC", "0")
    path, n = os.path.join(RSC, "anymal_c_like.urdf"), 128
    pb = _rsb_py.Batch(_rsb_py.Model(path), n, 0)
    bt = capi.Batch(capi.Model(path), n)
    gc = np.tile(ANYMAL_GC0.astype(np.float32), (n, 1)); gc[:, 2] = 0.54
    gc[:, 7:] += np.random.default_rng(9).uniform(-0.1, 0.1, (n, 12)).astype(np.float32)
    pb.set_ground(0.0); bt.set_ground(0.0)
    torch.from_dlpack(pb.gc()).copy_(torch.from_numpy(gc).cuda())
    bt.set_state(gc, np.zeros((n, 18), np.float32))
    body, pos, rot = _sensors(load_tables(path), np.random.default_rng(92))
    pb.set_imus(body.tolist(), pos.reshape(-1).tolist(), rot.reshape(-1).tolist()); bt.set_imus(body, pos, rot)
    torch.cuda.synchronize()
    pb.integrate(SUB); bt.integrate(SUB)
    tl, ta = torch.zeros((n, len(body), 3), device="cuda"), torch.zeros((n, len(body), 3), device="cuda")
    pb.imu_readings(tl.data_ptr(), ta.data_ptr()); pb.sync()
    lin, ang = bt.imu_readings()
    assert np.abs(lin).max() > 1.0 and tl.cpu().numpy().tobytes() == lin.tobytes() and ta.cpu().numpy().tobytes() == ang.tobytes()


def test_cpp_imu_example():
    """the raisim:: facade: setImus / getImuLinearAcceleration / getImuAngularVelocity inside VectorizedEnvironment (one launch per
    control step, a batch of 256 against a batch of one) and stand-alone (examples/imu.cpp)"""
    exe = os.path.join(ROOT, "examples", "imu")
    if not os.path.exists(exe):
        subprocess.check_call(["make", "-C", os.path.join(ROOT, "examples")])
    out = subprocess.run([exe, os.path.join(RSC, "anymal_c_like.urdf")], capture_output=True, text=True, timeout=300)
    print(out.stdout)
    assert out.returncode == 0, out.stdout + out.stderr
