"""Actuation delay (rsb_batch_set_actuation_delay / clear_actuation_delay) through the C-ABI on an H100 (pytest -m gpu), on the quadruped
instance on a height map, the humanoid instance on the ground and the generic instance with leg self-collision pairs: delays of 0 and no
delay agree bit for bit; a delayed batch equals an undelayed one fed the restated applied command of tests/actuation_delay_ref.py one
sub-step at a time (PD mode, force mode, an actuator network); launch shapes, partial resets, non-advancing launches, the command
sources, the gym task, refusals, the launch count and the C++ facade example."""
import os

import numpy as np
import pytest

from conftest import ROOT, RSC
from actuation_delay_ref import applied
from actuator_network_ref import random_layers
from test_gpu_actuator_params import SETUPS
from test_gpu_contact_forces import _make, _outputs, _same
from test_self_collision_oracle import anymal_leg_pairs

pytestmark = pytest.mark.gpu

SUB, DMAX = 4, 16


@pytest.fixture(scope="module")
def capi():
    import torch
    assert torch.cuda.is_available(), "GPU tests need a CUDA device"
    from raisimlib_b200 import capi as c
    assert c.ACTUATION_DELAY_MAX == DMAX
    return c


def _setup(capi, monkeypatch, which, n, seed, wpc=None, mode="pd"):
    """_make's robots with the leg pairs on the generic instance, contact forces on every body, and `mode` "pd", "force" or "network"
    (an actuator network on every joint); a delay is set by the caller"""
    case, terrain, pairs = SETUPS[which]
    c = _make(capi, monkeypatch, case, n, terrain, seed, wpc=wpc, oracles=False)
    bt, t = c["bt"], c["t"]
    if pairs:
        bt.set_self_collision(anymal_leg_pairs())
    if mode == "force":
        bt.set_control_mode(capi.FORCE_AND_TORQUE)
    if mode == "network":
        bt.set_actuator_network(np.arange(6, t["nv"]), random_layers(np.random.default_rng(seed + 2), 2, 2, 16), 2)
    bt.set_contact_bodies(list(range(min(t["nb"], 32))))
    return c


def _commands(c, steps, seed):
    """per control step: position targets [n, nq], velocity targets [n, nv] and feed-forward torques [n, nv] that change every step
    (the base part of the position target stays, the base velocity target and torque are 0)"""
    t, n = c["t"], c["n"]
    rng = np.random.default_rng(seed)
    out = []
    for _ in range(steps):
        pt = c["pt"].copy(); pt[:, 7:] += rng.uniform(-0.25, 0.25, (n, t["nq"] - 7)).astype(np.float32)
        vt = np.zeros((n, t["nv"]), np.float32); vt[:, 6:] = rng.uniform(-1.0, 1.0, (n, t["nv"] - 6))
        tau = np.zeros((n, t["nv"]), np.float32); tau[:, 6:] = rng.uniform(-8.0, 8.0, (n, t["nv"] - 6))
        out.append((pt, vt, tau))
    return out


def _outs(bt):
    o = _outputs(bt)
    o["f"], o["s"] = bt.body_contact_forces()
    return o


def _same_but_forces(a, b, what):
    """_same without the contact forces per body: they are means over the last launch, so launches of other lengths report others"""
    _same({k: v for k, v in a.items() if k not in ("f", "s")}, b, what)


def _drive(bt, cmds, shape=(1, SUB), between=None):
    """one control step per command: set it, then `shape` = (launches, sub-steps each); outputs after every control step"""
    out = []
    for k, (pt, vt, tau) in enumerate(cmds):
        bt.set_pd_target(pt, vt)
        bt.set_generalized_force(tau)
        for _ in range(shape[0]):
            bt.integrate(shape[1])
        out.append(_outs(bt))
        if between:
            between(k)
    return out


def _restated(bt, cmds, delay, empty_at=None):
    """an undelayed batch fed, one sub-step at a time, each environment's applied command: delay [n] in force from sub-step 0;
    empty_at: (sub-step, [n] new delay or -1) -- environments with an entry >= 0 empty their history there and take the new delay"""
    n, T = len(delay), len(cmds) * SUB
    d = np.tile(np.asarray(delay)[:, None], (1, T))
    emp = [set() for _ in range(n)]
    if empty_at is not None:
        s0, nd = empty_at
        for e in np.nonzero(np.asarray(nd) >= 0)[0]:
            emp[e].add(s0)
            d[e, s0:] = nd[e]
    per_sub = [np.repeat(np.stack([c[i] for c in cmds]), SUB, axis=0) for i in range(3)]   # [T, n, w]
    app = [np.empty_like(p) for p in per_sub]
    for e in range(n):
        for i in range(3):
            app[i][:, e] = applied(per_sub[i][:, e], d[e], emp[e])
    out = []
    for s in range(T):
        bt.set_pd_target(np.ascontiguousarray(app[0][s]), np.ascontiguousarray(app[1][s]))
        bt.set_generalized_force(np.ascontiguousarray(app[2][s]))
        bt.integrate(1)
        if s % SUB == SUB - 1:
            out.append(_outs(bt))
    return out


# ---- 1: off is off ---------------------------------------------------------------------------------------------------------------------

@pytest.mark.parametrize("which", list(SETUPS))
def test_no_delay_zero_delays_cleared_and_reset_to_zero_agree(capi, monkeypatch, which):
    n, steps = 300, 4
    runs = {}
    for mode in ("never", "zeros", "cleared", "zero_after_delayed"):
        c = _setup(capi, monkeypatch, which, n, seed=11)
        bt = c["bt"]
        cmds = _commands(c, steps, seed=12)
        if mode == "zeros":
            bt.set_actuation_delay(np.zeros(n, np.int32))
        elif mode == "cleared":
            bt.set_actuation_delay(np.random.default_rng(1).integers(0, DMAX + 1, n).astype(np.int32))
            bt.clear_actuation_delay()
        elif mode == "zero_after_delayed":
            bt.set_actuation_delay(np.random.default_rng(1).integers(1, DMAX + 1, n).astype(np.int32))
            _drive(bt, cmds[:2])
            bt.set_state(c["gc"], c["gv"])
            bt.set_actuation_delay(None)
        runs[mode] = _drive(bt, cmds)
    for mode in ("zeros", "cleared", "zero_after_delayed"):
        for k in range(steps):
            _same(runs["never"][k], runs[mode][k], f"{which} {mode}, control step {k}: ")


# ---- 2: shifted-command equivalence ----------------------------------------------------------------------------------------------------

CASES = [(w, m) for w in SETUPS for m in ("pd", "force")] + [("quadruped_hm", "network")]


@pytest.mark.parametrize("which,mode", CASES)
def test_delayed_batch_equals_an_undelayed_one_fed_the_restated_command(capi, monkeypatch, which, mode):
    """delays 0 .. 16 (longer than one 4-sub-step launch) against 1-sub-step launches fed cmd(max(t - d, 0)) for every environment;
    40 sub-steps, so that every delay runs past the kernel's counter wrap (t = 33 -> 17)"""
    n, steps = 204, 10
    delay = (np.arange(n) % (DMAX + 1)).astype(np.int32)
    a = _setup(capi, monkeypatch, which, n, seed=21, mode=mode)
    cmds = _commands(a, steps, seed=22)
    a["bt"].set_actuation_delay(delay)
    got = _drive(a["bt"], cmds)
    b = _setup(capi, monkeypatch, which, n, seed=21, mode=mode)
    want = _restated(b["bt"], cmds, delay)
    for k in range(steps):
        _same_but_forces(want[k], got[k], f"{which} {mode}, control step {k}: ")
    # the delay was seen: an undelayed batch fed the commanded rows ends elsewhere
    c = _setup(capi, monkeypatch, which, n, seed=21, mode=mode)
    plain = _drive(c["bt"], cmds)
    assert plain[-1]["gc"][delay > 0].tobytes() != got[-1]["gc"][delay > 0].tobytes()


# ---- 3: launch shapes ------------------------------------------------------------------------------------------------------------------

@pytest.mark.parametrize("which", list(SETUPS))
def test_launch_shapes_and_warps_per_cta_give_the_same_bits(capi, monkeypatch, which):
    n, steps = 200, 3
    delay = np.random.default_rng(3).integers(0, DMAX + 1, n).astype(np.int32)
    ref = None
    runs = [((1, 4), None), ((2, 2), None), ((4, 1), None)] + [((1, 4), w) for w in (28, 16, 14, 8, 4, 1)]
    for shape, wpc in runs:
        c = _setup(capi, monkeypatch, which, n, seed=31, wpc=wpc)
        c["bt"].set_actuation_delay(delay)
        out = _drive(c["bt"], _commands(c, steps, seed=32), shape=shape)
        if ref is None:
            ref = out
        else:
            for k in range(steps):
                (_same if shape == (1, SUB) else _same_but_forces)(ref[k], out[k], f"{which} shape {shape} wpc {wpc}, control step {k}: ")


# ---- 4: partial reset ------------------------------------------------------------------------------------------------------------------

@pytest.mark.parametrize("source", ["host", "device"])
def test_partial_reset(capi, monkeypatch, source):
    """after two control steps, a third of the environments get a new delay (their history restarts), the rest -1 (untouched)"""
    import torch
    n, steps, which = 240, 5, "quadruped_hm"
    rng = np.random.default_rng(4)
    delay = rng.integers(0, DMAX + 1, n).astype(np.int32)
    new = np.where(np.arange(n) % 3 == 0, rng.integers(0, DMAX + 1, n), -1).astype(np.int32)
    a = _setup(capi, monkeypatch, which, n, seed=41)
    cmds = _commands(a, steps, seed=42)
    a["bt"].set_actuation_delay(delay)

    def reset(k):
        if k == 1:
            if source == "host":   # two range calls: the second from env_begin
                a["bt"].set_actuation_delay(new[:n // 2])
                a["bt"].set_actuation_delay(new[n // 2:], env_begin=n // 2)
            else:
                a["bt"].set_actuation_delay_from(torch.from_numpy(new).cuda())
    got = _drive(a["bt"], cmds, between=reset)
    b = _setup(capi, monkeypatch, which, n, seed=41)
    want = _restated(b["bt"], cmds, delay, empty_at=(2 * SUB, new))
    for k in range(steps):
        _same_but_forces(want[k], got[k], f"{source}, control step {k}: ")
    # the -1 environments equal a run without the call
    c = _setup(capi, monkeypatch, which, n, seed=41)
    c["bt"].set_actuation_delay(delay)
    plain = _drive(c["bt"], cmds)
    keep = new < 0
    assert plain[-1]["gc"][keep].tobytes() == got[-1]["gc"][keep].tobytes()


# ---- 5: launches that do not advance the state -----------------------------------------------------------------------------------------

def test_non_advancing_launches_record_nothing(capi, monkeypatch):
    n, steps, which = 160, 3, "quadruped_hm"
    delay = np.random.default_rng(5).integers(0, DMAX + 1, n).astype(np.int32)
    runs = {}
    for mode in ("plain", "getters", "split"):
        c = _setup(capi, monkeypatch, which, n, seed=51)
        bt = c["bt"]
        bt.set_actuation_delay(delay)
        cmds = _commands(c, steps, seed=52)
        if mode == "plain":
            runs[mode] = _drive(bt, cmds, shape=(SUB, 1))
        elif mode == "getters":
            bt.set_frames([0], np.zeros((1, 3), np.float32))
            bt.set_height_scan([0, 0], np.array([[0.3, 0.0], [0.0, 0.3]], np.float32))

            def noise(k):
                bt.integrate1()
                bt.mass_matrix(); bt.nonlinearities(); bt.body_poses(); bt.update_kinematics()
                bt.frame_states(); bt.frame_jacobians(); bt.height_scan()
            runs[mode] = _drive(bt, cmds, shape=(SUB, 1), between=noise)
        else:   # integrate1 + integrate2 = integrate(1)
            out = []
            for pt, vt, tau in cmds:
                bt.set_pd_target(pt, vt); bt.set_generalized_force(tau)
                for _ in range(SUB):
                    bt.integrate1(); bt.integrate2()
                out.append(_outs(bt))
            runs[mode] = out
    for mode in ("getters", "split"):
        for k in range(steps):
            _same(runs["plain"][k], runs[mode][k], f"{mode}, control step {k}: ")


# ---- 6: command sources ----------------------------------------------------------------------------------------------------------------

def test_bound_and_pinned_targets_are_delayed_like_set_pd_target(capi, monkeypatch):
    import torch
    n, steps, which = 200, 4, "quadruped_hm"
    delay = np.random.default_rng(6).integers(0, DMAX + 1, n).astype(np.int32)
    runs = {}
    for mode in ("set", "bound", "control_step"):
        c = _setup(capi, monkeypatch, which, n, seed=61)
        bt = c["bt"]
        bt.set_actuation_delay(delay)
        cmds = [(pt, np.zeros_like(vt), tau) for pt, vt, tau in _commands(c, steps, seed=62)]
        if mode == "set":
            runs[mode] = _drive(bt, cmds)
            continue
        buf = torch.empty((n, c["t"]["nq"]), dtype=torch.float32, device="cuda")
        pin = torch.empty((n, c["t"]["nq"]), dtype=torch.float32).pin_memory()
        obs = np.empty((n, bt.ob_dim()), np.float32)
        if mode == "bound":
            bt.bind_pd_target(buf)
        out = []
        for pt, vt, tau in cmds:
            bt.set_generalized_force(tau)
            if mode == "bound":
                buf.copy_(torch.from_numpy(pt))
                bt.integrate(SUB)
            else:
                pin.copy_(torch.from_numpy(pt))
                bt.control_step(pin, SUB, obs)
            out.append(_outs(bt))
        runs[mode] = out
    for mode in ("bound", "control_step"):
        for k in range(steps):
            _same(runs["set"][k], runs[mode][k], f"{mode}, control step {k}: ")


def test_force_mode_in_place_targets_then_pd_mode_with_zero_delays(capi, monkeypatch):
    """force-mode control steps with pinned host targets, then PD mode: delays of 0 give the bits of no delay.  In force mode the targets
    go through the batch's own rows (no in-place read, no store from the kernel), so both batches enter PD mode with the same rows"""
    import torch
    n, steps, which = 200, 3, "quadruped_hm"
    runs = {}
    for mode in ("never", "zeros"):
        c = _setup(capi, monkeypatch, which, n, seed=65, mode="force")
        bt = c["bt"]
        if mode == "zeros":
            bt.set_actuation_delay(np.zeros(n, np.int32))
        cmds = _commands(c, 2 * steps, seed=66)
        pin = torch.empty((n, c["t"]["nq"]), dtype=torch.float32).pin_memory()
        obs = np.empty((n, bt.ob_dim()), np.float32)
        out = []
        for k, (pt, vt, tau) in enumerate(cmds):
            if k == steps:
                bt.set_control_mode(capi.PD_PLUS_FEEDFORWARD_TORQUE)
            bt.set_generalized_force(tau)
            if k < steps:
                pin.copy_(torch.from_numpy(pt))
                bt.control_step(pin, SUB, obs)
            else:
                bt.integrate(SUB)   # PD mode on the targets the force-mode steps left in the batch's rows
            out.append(_outs(bt))
        runs[mode] = out
    for k in range(2 * steps):
        _same(runs["never"][k], runs["zeros"][k], f"control step {k}: ")


def _gym(capi, monkeypatch, n, seed):
    c = _setup(capi, monkeypatch, "quadruped_hm", n, seed=seed)
    bt, t = c["bt"], c["t"]
    bt.gym_configure(c["gc"][0], np.zeros(t["nv"], np.float32), c["pt"][0, 7:], np.full(12, 0.5, np.float32), [3, 6])
    bt.gym_reset()
    return bt


def test_gym_step_equals_an_undelayed_gym_fed_the_shifted_actions(capi, monkeypatch):
    """delays 4k: the action of control step max(c - k, 0) since the last emptying, which every termination and gym_reset is"""
    n, steps = 256, 24
    k = (np.arange(n) % 4).astype(np.int64)
    a, b = _gym(capi, monkeypatch, n, 71), _gym(capi, monkeypatch, n, 71)
    a.set_actuation_delay((4 * k).astype(np.int32))
    rng = np.random.default_rng(72)
    shape = (n, a.ob_dim())
    oa, ob_ = np.empty(shape, np.float32), np.empty(shape, np.float32)
    ra, rb, da, db = np.empty(n, np.float32), np.empty(n, np.float32), np.empty(n, np.uint8), np.empty(n, np.uint8)
    hist = [[] for _ in range(n)]   # actions since the last emptying
    terminated = 0
    for s in range(steps):
        if s == 15:
            a.gym_reset(); b.gym_reset()
            hist = [[] for _ in range(n)]
        act = rng.uniform(-3, 3, (n, 12)).astype(np.float32)
        shifted = np.empty_like(act)
        for e in range(n):
            hist[e].append(act[e])
            shifted[e] = hist[e][max(len(hist[e]) - 1 - k[e], 0)]
        a.gym_step(act, SUB, oa, ra, da)
        b.gym_step(shifted, SUB, ob_, rb, db)
        assert oa.tobytes() == ob_.tobytes() and ra.tobytes() == rb.tobytes() and da.tobytes() == db.tobytes(), f"gym step {s}"
        for e in np.nonzero(da)[0]:
            hist[e] = []
        terminated += int(da.sum())
    print(f"{terminated} terminations over {steps} gym steps")
    assert terminated > 0


# ---- 7: refusals -----------------------------------------------------------------------------------------------------------------------

def test_refusals_change_nothing(capi, monkeypatch):
    import ctypes as C
    import torch
    n, which = 64, "quadruped_hm"
    delay = np.random.default_rng(8).integers(0, DMAX + 1, n).astype(np.int32)
    a, b = _setup(capi, monkeypatch, which, n, seed=81), _setup(capi, monkeypatch, which, n, seed=81)
    cmds = _commands(a, 4, seed=82)
    for bt in (a["bt"], b["bt"]):
        bt.set_actuation_delay(delay)
    _drive(a["bt"], cmds[:2]); _drive(b["bt"], cmds[:2])
    L_ = capi.lib()
    launches = a["bt"].launch_count()
    ok = np.zeros(n, np.int32)
    for eb, ec, wh in ((0, n + 1, capi.HOST), (-1, 2, capi.HOST), (0, -1, capi.HOST), (0, 2, 7)):
        assert L_.rsb_batch_set_actuation_delay(a["bt"].h, ok.ctypes.data_as(C.c_void_p), eb, ec, wh) == -1
    for v in (-2, DMAX + 1, -2**31, 2**31 - 1):
        bad = ok.copy(); bad[n - 1] = v
        with pytest.raises(capi.RsbError, match=f"environment {n - 1}"):
            a["bt"].set_actuation_delay(bad)
        with pytest.raises(capi.RsbError, match=f"environment {n - 1}"):
            a["bt"].set_actuation_delay_from(torch.from_numpy(bad).cuda())
    with pytest.raises(ValueError):
        a["bt"].set_actuation_delay_from(torch.zeros(n, dtype=torch.int64, device="cuda"))
    assert a["bt"].launch_count() == launches
    ga, gb = _drive(a["bt"], cmds[2:]), _drive(b["bt"], cmds[2:])
    for k in range(2):
        _same(gb[k], ga[k], f"after refusals, control step {k}: ")


# ---- 8: launches and the facade ------------------------------------------------------------------------------------------------------

def test_delays_add_no_launch(capi, monkeypatch):
    n = 256
    c = _setup(capi, monkeypatch, "quadruped_hm", n, seed=91)
    bt = c["bt"]
    bt.set_actuation_delay(np.random.default_rng(9).integers(0, DMAX + 1, n).astype(np.int32))
    obs = np.empty((n, bt.ob_dim()), np.float32)
    l0 = bt.launch_count()
    for _ in range(5):
        bt.control_step(c["pt"], SUB, obs)
    assert bt.launch_count() - l0 == 5


def test_cpp_actuation_delay_example():
    """the facade example (examples/actuation_delay.cpp): one launch per control step, delays drawn in reset(), and environments bit for
    bit equal to stand-alone Worlds fed the shifted targets"""
    import subprocess
    exe = os.path.join(ROOT, "examples", "actuation_delay")
    if not os.path.exists(exe):
        subprocess.check_call(["make", "-C", os.path.join(ROOT, "examples")])
    out = subprocess.run([exe, os.path.join(RSC, "anymal_c_like.urdf")], capture_output=True, text=True, timeout=600)
    print(out.stdout)
    assert out.returncode == 0, out.stdout + out.stderr
    assert "launches per control step 1.00" in out.stdout
    assert ", 0 differ" in out.stdout
