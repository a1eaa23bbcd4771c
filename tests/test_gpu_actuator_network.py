"""Learned actuator network (rsb_batch_set_actuator_network / set_actuator_history / get_actuator_history) through the C-ABI on an H100
(pytest -m gpu), on the quadruped instance on a height map, the humanoid instance on the ground and the generic instance with leg
self-collision pairs: the torque against the float64 restatement of tests/actuator_network_ref.py and the history shift bit for bit,
the dynamics against the float64 oracle driven by the restated torque, invariance (launch shapes, warps per CTA, set then cleared,
launches that must not shift the history, force mode), saturation, resets, refusals, the launch count and the C++ facade example."""
import os

import numpy as np
import pytest

from conftest import ROOT, RSC
from actuator_network_ref import features, net, random_layers, shift, torque
from test_gpu_actuator_params import SETUPS, _limits
from test_gpu_contact_forces import _make, _outputs, _same
from test_self_collision_oracle import anymal_leg_pairs

pytestmark = pytest.mark.gpu

SUB, H, L, W = 4, 3, 3, 32


@pytest.fixture(scope="module")
def capi():
    import torch
    assert torch.cuda.is_available(), "GPU tests need a CUDA device"
    from raisimlib_b200 import capi as c
    return c


def _setup(capi, monkeypatch, which, n, seed, wpc=None, oracles=False, history=H, layers=L, width=W, network=True):
    """_make's robots (PD mode, gains and targets set) with random feed-forward torques, targets further away, the leg pairs on the
    generic instance, and a seeded network on every joint dof"""
    case, terrain, pairs = SETUPS[which]
    c = _make(capi, monkeypatch, case, n, terrain, seed, wpc=wpc, oracles=oracles)
    t, bt = c["t"], c["bt"]
    rng = np.random.default_rng(seed + 1)
    pt = c["pt"].copy(); pt[:, 7:] += rng.uniform(-0.3, 0.3, (n, t["nq"] - 7)).astype(np.float32)
    bt.set_pd_target(pt, np.zeros((n, t["nv"]), np.float32))
    tau = np.zeros((n, t["nv"]), np.float32); tau[:, 6:] = rng.uniform(-5.0, 5.0, (n, t["nv"] - 6))
    bt.set_generalized_force(tau)
    if pairs:
        bt.set_self_collision(anymal_leg_pairs())
    c.update(pt=pt, tau=tau, dofs=np.arange(6, t["nv"]), layers=random_layers(np.random.default_rng(seed + 2), history, layers, width))
    if network:
        bt.set_actuator_network(c["dofs"], c["layers"], history)
    return c


def _random_history(rng, n, nd, history):
    return np.concatenate([rng.uniform(-0.4, 0.4, (n, nd, 1, history - 1)), rng.uniform(-3.0, 3.0, (n, nd, 1, history - 1))], axis=2).astype(np.float32)


def _ev(c, gc, gv, pt):
    """this sub-step's (e, v) of every listed dof from float32 rows: the kernel's float32 subtraction"""
    t, d = c["t"], c["dofs"]
    qmap = {t["vidx"][b]: t["qidx"][b] for b in range(1, t["nb"])}
    q = np.array([qmap[i] for i in d])
    return pt[:, q] - gc[:, q], gv[:, d]


# ---- 1: torque accuracy and the history shift -----------------------------------------------------------------------------------------

@pytest.mark.parametrize("which", list(SETUPS))
def test_torque_matches_the_restatement_and_history_shifts_bit_for_bit(capi, monkeypatch, which):
    n = 512
    c = _setup(capi, monkeypatch, which, n, seed=11)
    bt, t, d = c["bt"], c["t"], c["dofs"]
    rows = _random_history(np.random.default_rng(5), n, len(d), H)
    bt.set_actuator_history(rows)
    assert bt.actuator_history().tobytes() == rows.tobytes()
    gc, gv = bt.get_state()
    bt.integrate(1)
    e, v = _ev(c, gc, gv, c["pt"])
    lim = _limits(t)[d]
    ref = torque(c["layers"], e, v, rows, c["tau"][:, d], lim)
    got = bt.generalized_force()[:, d]
    err = np.abs(got - ref) / (1.0 + np.abs(ref))
    sat = np.abs(np.abs(ref) - lim) < 1e-9
    print(f"{which}: {len(d)} dofs, |tau| median {np.median(np.abs(ref)):.2f}, {int(sat.sum())} saturated, max rel err {err.max():.2e}")
    assert err.max() <= 1e-4
    assert np.abs(ref).max() > 5.0
    assert bt.actuator_history().tobytes() == shift(e, v, rows).tobytes()


# ---- 2: dynamics against the oracle ---------------------------------------------------------------------------------------------------

@pytest.mark.parametrize("which", list(SETUPS))
def test_dynamics_match_the_oracle_driven_by_the_restated_torque(capi, monkeypatch, which):
    """20 sub-steps one launch at a time.  The float64 and float32 oracles (with the leg pairs on the generic instance) run each with
    tau_ff = the restated torque from their own state and history and no PD law on the listed dofs.  The kernel stays within the
    per-environment gain test's bounds of the float64 oracle, or within a few times the float32 oracle's own distance from it, as the
    parity tests bound the kernel where float32 rounding is amplified (the humanoid's 30 network joints)"""
    n = 256
    c = _setup(capi, monkeypatch, which, n, seed=21, oracles=True)
    bt, t, d = c["bt"], c["t"], c["dofs"]
    oracles = c["o"]
    if SETUPS[which][2]:   # the oracle with self-collision pairs, on _make's height map (its first draw from the seed)
        from oracle.self_oracle import SelfOracle
        hm = (0.1 * np.random.default_rng(21).uniform(-1, 1, (49, 65))).astype(np.float32)
        oracles = [SelfOracle(t, params=dict(threshold=1e-6)), SelfOracle(t, precision="f32", params=dict(threshold=1e-6))]
        for o in oracles:
            o.set_heightmap(65, 49, 12.8, 9.6, 0.1, -0.2, hm.astype(np.float64))
            o.set_self_collision(anymal_leg_pairs())
    kp, kd = c["kp"].copy(), c["kd"].copy(); kp[d] = 0.0; kd[d] = 0.0
    lim = _limits(t)[d]
    pt64 = c["pt"].astype(np.float64)
    sides = [dict(o=o, a=c["gc"].astype(np.float64), b=c["gv"].astype(np.float64), hist=np.zeros((n, len(d), 2, H - 1)),
                  status=np.zeros(n, np.int32)) for o in oracles]
    for k in range(20):
        bt.integrate(1)
        for sd in sides:
            e, v = _ev(c, sd["a"], sd["b"], pt64)
            tau = c["tau"].astype(np.float64).copy()
            tau[:, d] = torque(c["layers"], e, v, sd["hist"], tau[:, d], lim)
            sd["hist"] = shift(e, v, sd["hist"])
            dd = sd["o"].step(sd["a"], sd["b"], tau_ff=tau, ptarget=pt64, vtarget=np.zeros((n, t["nv"])), kp=kp, kd=kd, debug=True)
            sd["status"] = dd["status"]
    g, _ = bt.get_state()
    conv = (bt.solver_status() <= 1) & (sides[0]["status"] <= 1) & (sides[1]["status"] <= 1)
    eg = np.abs(g - sides[0]["a"]).max(1)[conv]
    e32 = np.abs(sides[1]["a"] - sides[0]["a"]).max(1)[conv]
    print(f"{which}: 20 sub-steps ({int(conv.sum())} converged): median |dgc| {np.median(eg):.2e} p90 {np.quantile(eg, 0.9):.2e}; "
          f"f32 oracle median {np.median(e32):.2e} p90 {np.quantile(e32, 0.9):.2e}")
    assert conv.mean() > 0.8
    assert np.median(eg) < max(2e-5, 3 * np.median(e32))
    assert np.quantile(eg, 0.9) < max(2e-4, 3 * np.quantile(e32, 0.9))


# ---- 3: invariance -------------------------------------------------------------------------------------------------------------------

def _run(bt, shape, steps=3):
    out = []
    for _ in range(steps):
        if shape == "one":
            bt.integrate(SUB)
        else:
            for _ in range(SUB):
                bt.integrate(1)
        o = _outputs(bt)
        o["hist"] = bt.actuator_history()
        out.append(o)
    return out


@pytest.mark.parametrize("which", list(SETUPS))
def test_one_launch_of_four_equals_four_launches_of_one(capi, monkeypatch, which):
    runs = {}
    for shape in ("one", "four"):
        c = _setup(capi, monkeypatch, which, 300, seed=31)
        runs[shape] = _run(c["bt"], shape)
    for k in range(3):
        _same(runs["one"][k], runs["four"][k], f"{which} control step {k}: ")


@pytest.mark.parametrize("which", list(SETUPS))
def test_every_warps_per_cta_choice_gives_the_same_bits(capi, monkeypatch, which):
    ref = None
    for wpc in (28, 16, 14, 8, 4, 1):
        c = _setup(capi, monkeypatch, which, 200, seed=41, wpc=wpc)
        out = _run(c["bt"], "one", steps=2)
        if ref is None:
            ref = out
        else:
            for k in range(2):
                _same(ref[k], out[k], f"{which} wpc {wpc}, control step {k}: ")


@pytest.mark.parametrize("which", list(SETUPS))
def test_set_then_cleared_equals_never_set(capi, monkeypatch, which):
    runs = {}
    for mode in ("never", "cleared"):
        c = _setup(capi, monkeypatch, which, 300, seed=51, network=mode == "cleared")
        bt = c["bt"]
        if mode == "cleared":
            bt.integrate(SUB); bt.set_state(c["gc"], c["gv"])
            bt.set_actuator_network([], None, H)
        bt.set_contact_bodies(list(range(min(c["t"]["nb"], 32))))
        runs[mode] = []
        for _ in range(4):
            bt.integrate(SUB)
            o = _outputs(bt)
            o["f"], o["s"] = bt.body_contact_forces()
            runs[mode].append(o)
    for k in range(4):
        _same(runs["never"][k], runs["cleared"][k], f"{which} control step {k}: ")


def test_only_advancing_launches_shift_the_history(capi, monkeypatch):
    """integrate1, the getters, the kinematics pass and the height scan leave it; integrate2 shifts it once; force mode leaves it and
    applies tau_ff to the listed dofs"""
    n = 128
    c = _setup(capi, monkeypatch, "quadruped_hm", n, seed=61)
    bt, d = c["bt"], c["dofs"]
    rows = _random_history(np.random.default_rng(6), n, len(d), H)
    bt.set_actuator_history(rows)
    bt.integrate1()
    bt.mass_matrix(); bt.nonlinearities(); bt.body_poses(); bt.update_kinematics()
    bt.set_frames([0], np.zeros((1, 3), np.float32)); bt.frame_states(); bt.frame_jacobians()
    bt.set_height_scan([0, 0], np.array([[0.3, 0.0], [0.0, 0.3]], np.float32)); bt.height_scan()
    assert bt.actuator_history().tobytes() == rows.tobytes()
    gc, gv = bt.get_state()
    bt.integrate2()
    e, v = _ev(c, gc, gv, c["pt"])
    assert bt.actuator_history().tobytes() == shift(e, v, rows).tobytes()
    # force mode: history untouched, tau_ff applied (saturated) on the listed dofs
    bt.set_actuator_history(rows)
    bt.set_control_mode(capi.FORCE_AND_TORQUE)
    bt.integrate(SUB)
    assert bt.actuator_history().tobytes() == rows.tobytes()
    lim = _limits(c["t"])[d]
    assert np.array_equal(bt.generalized_force()[:, d], np.clip(c["tau"][:, d], -lim, lim))


# ---- 4: saturation ---------------------------------------------------------------------------------------------------------------------

def test_urdf_and_per_environment_effort_limits_clamp_the_network(capi, monkeypatch):
    n = 256
    c = _setup(capi, monkeypatch, "quadruped_hm", n, seed=71)
    bt, t, d = c["bt"], c["t"], c["dofs"]
    # a network with large outputs: many dofs reach the URDF limit
    big = [(w, b) for w, b in c["layers"][:-1]] + [(c["layers"][-1][0] * 20.0, c["layers"][-1][1])]
    bt.set_actuator_network(d, big, H)
    gc, gv = bt.get_state()
    bt.integrate(1)
    e, v = _ev(c, gc, gv, c["pt"])
    zero = np.zeros((n, len(d), 2, H - 1))
    lim = _limits(t)[d]
    free = c["tau"][:, d] + net(big, features(e, v, zero))
    got = bt.generalized_force()[:, d]
    over = np.abs(free) > lim * 1.001
    assert over.mean() > 0.1
    assert np.array_equal(got[over], (np.sign(free[over]) * lim[np.nonzero(over)[1]]).astype(np.float32))
    assert np.abs(got).max() <= lim.max()
    # per-environment effort rows: every environment its own limit
    rows = np.full((n, t["nv"], 3), -1.0, np.float32)
    elim = np.random.default_rng(7).uniform(2.0, 30.0, (n, 1)).astype(np.float32)
    rows[:, 6:, 2] = elim
    bt.set_actuator_params(rows)
    bt.set_actuator_network(d, big, H)
    gc, gv = bt.get_state()
    bt.integrate(1)
    e, v = _ev(c, gc, gv, c["pt"])
    free = c["tau"][:, d] + net(big, features(e, v, zero))
    got = bt.generalized_force()[:, d]
    over = np.abs(free) > elim * 1.001
    assert over.mean() > 0.3
    assert np.array_equal(got[over], (np.sign(free) * elim)[over].astype(np.float32))
    assert (np.abs(got) <= elim).all()


# ---- 5: resets -------------------------------------------------------------------------------------------------------------------------

def test_resets(capi, monkeypatch):
    n = 256
    c = _setup(capi, monkeypatch, "quadruped_hm", n, seed=81)
    bt, d = c["bt"], c["dofs"]
    zeros = np.zeros((n, len(d), 2, H - 1), np.float32)
    assert bt.actuator_history().tobytes() == zeros.tobytes()          # set zeroes
    bt.integrate(SUB)
    assert np.abs(bt.actuator_history()).max() > 0
    bt.set_actuator_network(d, c["layers"], H)
    assert bt.actuator_history().tobytes() == zeros.tobytes()
    bt.integrate(SUB)
    bt.set_actuator_history(None, 10, 20)                              # NULL zeroes the range only
    h = bt.actuator_history()
    assert not h[10:30].any() and h[:10].any() and h[30:].any()
    before = bt.actuator_history()
    bt.set_state(c["gc"], c["gv"])                                      # set_state keeps it
    assert bt.actuator_history().tobytes() == before.tobytes()
    # a sparse reset from torch stays on the device
    import torch
    ht = torch.empty((n, len(d), 2, H - 1), dtype=torch.float32, device="cuda")
    bt.actuator_history_into(ht)
    ht[torch.arange(0, n, 3, device="cuda")] = 0.0
    bt.set_actuator_history_from(ht)
    want = before.copy(); want[::3] = 0.0
    assert bt.actuator_history().tobytes() == want.tobytes()
    # gym reset zeroes all; gym-step terminations zero exactly the terminated environments
    t = c["t"]
    feet = [3, 6]   # contacts on two of the four shanks do not terminate: a mix of terminated and running environments
    bt.gym_configure(c["gc"][0], np.zeros(t["nv"], np.float32), c["pt"][0, 7:], np.full(12, 0.5, np.float32), feet)
    bt.gym_reset()
    assert bt.actuator_history().tobytes() == zeros.tobytes()
    bt.set_state(c["gc"], c["gv"])
    rng = np.random.default_rng(8)
    obs, rew, done = np.empty((n, bt.ob_dim()), np.float32), np.empty(n, np.float32), np.empty(n, np.uint8)
    terminated = 0
    for k in range(30):
        bt.gym_step(rng.uniform(-3, 3, (n, 12)).astype(np.float32), SUB, obs, rew, done)
        h = bt.actuator_history()
        assert not h[done == 1].any()
        assert (np.abs(h[done == 0]).reshape(int((done == 0).sum()), -1).max(1) > 0).all()
        terminated += int(done.sum())
    print(f"{terminated} terminations over 30 gym steps")
    assert terminated > 0


# ---- 6: refusals -----------------------------------------------------------------------------------------------------------------------

def test_refusals_change_nothing(capi, monkeypatch):
    import ctypes as C
    n = 64
    c = _setup(capi, monkeypatch, "quadruped_hm", n, seed=91)
    bt, d = c["bt"], c["dofs"]
    L_ = capi.lib()
    bt.integrate(SUB)
    hist0 = bt.actuator_history()

    def after():
        return bt.actuator_history()

    params = np.concatenate([np.concatenate([w.ravel(), b.ravel()]) for w, b in c["layers"]]).astype(np.float32)
    P = params.ctypes.data_as(C.c_void_p)
    dofs = np.ascontiguousarray(d, np.int32)

    def call(dl, nd, h=H, l=L, w=W, p=P):
        arr = np.ascontiguousarray(dl, np.int32)
        return L_.rsb_batch_set_actuator_network(bt.h, arr.ctypes.data_as(C.c_void_p) if len(arr) else None, nd, h, l, w, p)
    bad_nan = params.copy(); bad_nan[17] = np.nan
    bad_inf = params.copy(); bad_inf[-1] = np.inf
    cases = [(dofs, -1), (dofs, 19), (np.r_[dofs[:-1], 18], 12), (np.r_[dofs[:-1], -1], 12), (np.r_[dofs[:-1], 6], 12), (np.r_[dofs[:-1], 3], 12)]
    for dl, nd in cases:
        assert call(dl, nd) == -1
        assert after().tobytes() == hist0.tobytes()
    for kw in (dict(h=0), dict(h=5), dict(l=0), dict(l=5), dict(w=0), dict(w=33), dict(p=None),
               dict(p=bad_nan.ctypes.data_as(C.c_void_p)), dict(p=bad_inf.ctypes.data_as(C.c_void_p))):
        assert call(dofs, 12, **kw) == -1, kw
        assert after().tobytes() == hist0.tobytes()
    assert L_.rsb_batch_set_actuator_network(bt.h, None, 12, H, L, W, P) == -1
    # history calls: bad range, bad where, non-finite rows
    rows = np.zeros((n, len(d), 2, H - 1), np.float32)
    for eb, ec, wh in ((0, n + 1, capi.HOST), (-1, 2, capi.HOST), (0, 2, 7)):
        assert L_.rsb_batch_set_actuator_history(bt.h, rows.ctypes.data_as(C.c_void_p), eb, ec, wh) == -1
        assert L_.rsb_batch_get_actuator_history(bt.h, rows.ctypes.data_as(C.c_void_p), eb, ec, wh) == -1
    for v in (np.nan, np.inf, -np.inf):
        r = np.random.default_rng(9).uniform(-1, 1, rows.shape).astype(np.float32); r[n - 1, 3, 1, 1] = v
        with pytest.raises(capi.RsbError, match="not finite"):
            bt.set_actuator_history(r)
        assert after().tobytes() == hist0.tobytes()
    # the same steps as a twin that never saw a refusal
    c2 = _setup(capi, monkeypatch, "quadruped_hm", n, seed=91)
    c2["bt"].integrate(SUB)
    bt.integrate(SUB); c2["bt"].integrate(SUB)
    _same(_outputs(bt), _outputs(c2["bt"]), "after refusals: ")
    assert bt.actuator_history().tobytes() == c2["bt"].actuator_history().tobytes()
    # no network: the history calls are refused
    bt.set_actuator_network([], None, H)
    assert L_.rsb_batch_get_actuator_history(bt.h, rows.ctypes.data_as(C.c_void_p), 0, 1, capi.HOST) == -1
    assert b"no actuator network" in L_.rsb_last_error()
    # H = 1: rows of no words, both calls succeed
    bt.set_actuator_network(d, random_layers(np.random.default_rng(3), 1, 2, 8), 1)
    assert bt.actuator_history().shape == (n, len(d), 2, 0)
    bt.set_actuator_history(np.zeros((n, len(d), 2, 0), np.float32))
    bt.integrate(SUB)


# ---- 7: launches and gym acceptance ------------------------------------------------------------------------------------------------

def test_one_launch_per_control_step_and_gym_step(capi, monkeypatch):
    n = 256
    c = _setup(capi, monkeypatch, "quadruped_hm", n, seed=101)
    bt, t = c["bt"], c["t"]
    obs = np.empty((n, bt.ob_dim()), np.float32)
    l0 = bt.launch_count()
    for _ in range(5):
        bt.control_step(c["pt"], SUB, obs)
    assert bt.launch_count() - l0 == 5
    # a network alone (no gains, no rows) lets the gym task run: unlisted dofs have no PD law
    case, terrain, _ = SETUPS["quadruped_hm"]
    c2 = _make(capi, monkeypatch, case, n, terrain, 102, oracles=False)
    b2 = capi.Batch(capi.Model(os.path.join(RSC, "anymal_c_like.urdf")), n)
    b2.set_ground(0.0)
    b2.set_state(c2["gc"], c2["gv"])
    b2.set_actuator_network(c["dofs"], c["layers"], H)
    b2.gym_configure(c2["gc"][0], np.zeros(t["nv"], np.float32), c2["pt"][0, 7:], np.full(12, 0.5, np.float32), [])
    rew, done = np.empty(n, np.float32), np.empty(n, np.uint8)
    l0 = b2.launch_count()
    for _ in range(5):
        b2.gym_step(np.zeros((n, 12), np.float32), SUB, obs, rew, done)
    assert b2.launch_count() - l0 == 5
    assert np.isfinite(obs).all()


def test_cpp_actuator_network_example():
    """the facade example (examples/actuator_network.cpp): one launch per control step, resets through resetActuatorHistory, and
    getGeneralizedForce against a float64 restatement of the network"""
    import subprocess
    exe = os.path.join(ROOT, "examples", "actuator_network")
    if not os.path.exists(exe):
        subprocess.check_call(["make", "-C", os.path.join(ROOT, "examples")])
    out = subprocess.run([exe, os.path.join(RSC, "anymal_c_like.urdf")], capture_output=True, text=True, timeout=600)
    print(out.stdout)
    assert out.returncode == 0, out.stdout + out.stderr
    assert "launches per control step 1.00" in out.stdout
