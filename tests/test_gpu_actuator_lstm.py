"""LSTM actuator network (rsb_batch_set_actuator_lstm, its state through rsb_batch_{set,get}_actuator_history) through the C-ABI on an
H100 (pytest -m gpu), on the quadruped instance on a height map, the humanoid instance on the ground and the generic instance with leg
self-collision pairs: torque and (h, c) rows against the float64 restatement of tests/actuator_lstm_ref.py and against torch.nn.LSTM,
the dynamics against the float64 oracle driven by the restated torque, bit identity (launch shapes, warps per CTA, cleared, replaced by
the MLP, batch size), the state rules (advancing launches, force mode, effort limits, actuation delay, resets, round trips, non-finite
rows), refusals, the launch count, every per-environment feature at once, the pybind module and the C++ facade example."""
import ctypes as C
import os
import subprocess

import numpy as np
import pytest

from conftest import ROOT, RSC
from actuator_lstm_ref import count, flat, net, random_lstm, torque
from actuator_network_ref import random_layers
from test_gpu_actuator_network import _ev
from test_gpu_actuator_params import SETUPS, _limits
from test_gpu_contact_forces import _make, _outputs, _same
from test_gpu_feature_mix import _batch as _mix_batch, _command as _mix_command, _inputs as _mix_inputs, _wrench as _mix_wrench
from test_self_collision_oracle import anymal_leg_pairs

pytestmark = pytest.mark.gpu

SUB, L, HID = 4, 2, 8
REL = 1e-4          # |got - ref| / (1 + |ref|), the MLP test's bound


@pytest.fixture(scope="module")
def capi():
    import torch
    assert torch.cuda.is_available(), "GPU tests need a CUDA device"
    from raisimlib_b200 import capi as c
    return c


def _setup(capi, monkeypatch, which, n, seed, wpc=None, oracles=False, layers=L, hidden=HID, network=True):
    """_make's robots (PD mode, gains and targets set) with random feed-forward torques, targets further away, the leg pairs on the
    generic instance, and a seeded LSTM on every joint dof"""
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
    lp, ro = random_lstm(np.random.default_rng(seed + 2), layers, hidden)
    c.update(pt=pt, tau=tau, dofs=np.arange(6, t["nv"]), lstm=(lp, ro))
    if network:
        bt.set_actuator_lstm(c["dofs"], lp, ro)
    return c


def _random_state(rng, n, nd, layers=L, hidden=HID):
    s = rng.uniform(-0.8, 0.8, (n, nd, layers, 2, hidden))
    s[:, :, :, 1] *= 3.0
    return s.astype(np.float32)


def _rel(got, ref):
    return (np.abs(np.asarray(got, np.float64) - ref) / (1.0 + np.abs(ref))).max()


# ---- 1: accuracy ------------------------------------------------------------------------------------------------------------------------

@pytest.mark.parametrize("which", list(SETUPS))
def test_every_sub_step_matches_the_restatement(capi, monkeypatch, which):
    """4 launches of one sub-step from random (h, c) rows: the applied torque and the new rows of every sub-step against the restatement
    fed the float32 (e, v) of the GPU's own state and its own rows before the sub-step"""
    n = 512
    c = _setup(capi, monkeypatch, which, n, seed=11)
    bt, t, d = c["bt"], c["t"], c["dofs"]
    rows = _random_state(np.random.default_rng(5), n, len(d))
    bt.set_actuator_history(rows)
    assert bt.actuator_history().tobytes() == rows.tobytes()
    lim = _limits(t)[d]
    worst_t = worst_s = 0.0
    for k in range(SUB):
        gc, gv = bt.get_state()
        before = bt.actuator_history()
        bt.integrate(1)
        e, v = _ev(c, gc, gv, c["pt"])
        ref, state = torque(*c["lstm"], e, v, before, c["tau"][:, d], lim)
        worst_t = max(worst_t, _rel(bt.generalized_force()[:, d], ref))
        worst_s = max(worst_s, _rel(bt.actuator_history(), state))
        if k == 0:
            assert np.abs(ref).max() > 5.0
    print(f"{which}: {len(d)} dofs, 4 sub-steps: max rel err torque {worst_t:.2e}, (h, c) {worst_s:.2e}")
    assert worst_t <= REL and worst_s <= REL


def test_forty_launches_match_torch_lstm(capi, monkeypatch):
    """40 single-sub-step launches from zero state; the recorded (e, v) sequence through a float64 torch.nn.LSTM + nn.Linear: the net
    torque of every unsaturated dof at every step and the final (h, c) rows"""
    import torch
    n = 128
    c = _setup(capi, monkeypatch, "quadruped_hm", n, seed=13)
    bt, t, d = c["bt"], c["t"], c["dofs"]
    lp, ro = c["lstm"]
    lim = _limits(t)[d]
    xs, nets = [], []
    for _ in range(40):
        gc, gv = bt.get_state()
        bt.integrate(1)
        e, v = _ev(c, gc, gv, c["pt"])
        xs.append(np.stack([e, v], -1).astype(np.float64))
        nets.append(bt.generalized_force()[:, d].astype(np.float64) - c["tau"][:, d])
    lstm = torch.nn.LSTM(2, HID, L).double()
    lin = torch.nn.Linear(HID, 1).double()
    with torch.no_grad():
        for l, p in enumerate(lp):
            for name, a in zip(("weight_ih", "weight_hh", "bias_ih", "bias_hh"), p):
                getattr(lstm, f"{name}_l{l}").copy_(torch.from_numpy(a.astype(np.float64)))
        lin.weight.copy_(torch.from_numpy(ro[0].astype(np.float64))); lin.bias.copy_(torch.from_numpy(ro[1].astype(np.float64)))
        seq = torch.from_numpy(np.stack(xs).reshape(40, n * len(d), 2))
        out, (hT, cT) = lstm(seq)
        want = lin(out)[..., 0].numpy().reshape(40, n, len(d))
    got = np.stack(nets)
    free = np.abs(got + c["tau"][:, d]) < lim * 0.999          # not saturated: generalized force = tau_ff + net
    err = np.abs(got - want) / (1.0 + np.abs(want))
    hist = bt.actuator_history().astype(np.float64)             # [n, dofs, L, 2, HID]
    eh = _rel(hist[:, :, :, 0].reshape(n * len(d), L, HID).transpose(1, 0, 2), hT.numpy())
    ec = _rel(hist[:, :, :, 1].reshape(n * len(d), L, HID).transpose(1, 0, 2), cT.numpy())
    print(f"40 launches: {free.mean():.2f} of the torques unsaturated, max rel err net {err[free].max():.2e}, h {eh:.2e}, c {ec:.2e}")
    assert free.mean() > 0.5 and err[free].max() <= REL and eh <= REL and ec <= REL


@pytest.mark.parametrize("which", list(SETUPS))
def test_dynamics_match_the_oracle_driven_by_the_restated_torque(capi, monkeypatch, which):
    """20 sub-steps one launch at a time; the float64 and float32 oracles run each with tau_ff = the restated torque from their own state
    and (h, c) and no PD law on the listed dofs, under the bounds of the MLP's test"""
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
    sides = [dict(o=o, a=c["gc"].astype(np.float64), b=c["gv"].astype(np.float64), st=np.zeros((n, len(d), L, 2, HID)),
                  status=np.zeros(n, np.int32)) for o in oracles]
    for k in range(20):
        bt.integrate(1)
        for sd in sides:
            e, v = _ev(c, sd["a"], sd["b"], pt64)
            tau = c["tau"].astype(np.float64).copy()
            tau[:, d], sd["st"] = torque(*c["lstm"], e, v, sd["st"], tau[:, d], lim)
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


# ---- 2: bit identity ---------------------------------------------------------------------------------------------------------------

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
        c = _setup(capi, monkeypatch, which, 200, seed=41, wpc=wpc, hidden=32 if which == "quadruped_hm" else HID)
        out = _run(c["bt"], "one", steps=2)
        if ref is None:
            ref = out
        else:
            for k in range(2):
                _same(ref[k], out[k], f"{which} wpc {wpc}, control step {k}: ")


@pytest.mark.parametrize("clear_by", ["lstm", "mlp"])
@pytest.mark.parametrize("which", list(SETUPS))
def test_set_then_cleared_equals_never_set(capi, monkeypatch, which, clear_by):
    runs = {}
    for mode in ("never", "cleared"):
        c = _setup(capi, monkeypatch, which, 300, seed=51, network=mode == "cleared")
        bt = c["bt"]
        if mode == "cleared":
            bt.integrate(SUB); bt.set_state(c["gc"], c["gv"])
            if clear_by == "lstm":
                bt.set_actuator_lstm([], None, None)
            else:
                bt.set_actuator_network([], None, 1)
        bt.set_contact_bodies(list(range(min(c["t"]["nb"], 32))))
        runs[mode] = []
        for _ in range(4):
            bt.integrate(SUB)
            o = _outputs(bt)
            o["f"], o["s"] = bt.body_contact_forces()
            runs[mode].append(o)
    for k in range(4):
        _same(runs["never"][k], runs["cleared"][k], f"{which} control step {k}: ")


def test_lstm_replaced_by_the_mlp_equals_the_mlp_alone(capi, monkeypatch):
    layers = random_layers(np.random.default_rng(7), 3, 2, 16)
    runs = {}
    for mode in ("mlp", "replaced"):
        c = _setup(capi, monkeypatch, "quadruped_hm", 256, seed=55, network=mode == "replaced")
        bt = c["bt"]
        if mode == "replaced":
            bt.integrate(SUB); bt.set_state(c["gc"], c["gv"])
        bt.set_actuator_network(c["dofs"], layers, 3)
        runs[mode] = _run(bt, "one")
    for k in range(3):
        _same(runs["mlp"][k], runs["replaced"][k], f"control step {k}: ")
    assert runs["mlp"][0]["hist"].shape == (256, 12, 2, 2)


def test_a_batch_of_256_equals_batches_of_one(capi, monkeypatch):
    c = _setup(capi, monkeypatch, "quadruped_hm", 256, seed=57)
    big = _run(c["bt"], "one", steps=2)
    for e in (0, 101, 255):
        one = _make(capi, monkeypatch, "quadruped", 1, "hm", seed=57, oracles=False)
        b1 = one["bt"]
        b1.set_pd_target(c["pt"][e:e + 1], np.zeros((1, 18), np.float32))
        b1.set_generalized_force(c["tau"][e:e + 1])
        b1.set_state(c["gc"][e:e + 1], c["gv"][e:e + 1])
        b1.set_actuator_lstm(c["dofs"], *c["lstm"])
        small = _run(b1, "one", steps=2)
        for k in range(2):
            for key in ("gc", "gv", "tau", "hist"):
                assert np.asarray(small[k][key]).tobytes() == np.asarray(big[k][key])[e:e + 1].tobytes(), f"environment {e} step {k} {key}"


# ---- 3: state rules ---------------------------------------------------------------------------------------------------------------------

def test_only_advancing_launches_advance_the_state(capi, monkeypatch):
    """integrate1, the getters, the kinematics pass and the height scan leave it; integrate2 advances it once; control_step once per
    sub-step; force mode leaves it and applies tau_ff to the listed dofs"""
    n = 128
    c = _setup(capi, monkeypatch, "quadruped_hm", n, seed=61)
    bt, d = c["bt"], c["dofs"]
    lim = _limits(c["t"])[d]
    rows = _random_state(np.random.default_rng(6), n, len(d))
    bt.set_actuator_history(rows)
    bt.integrate1()
    bt.mass_matrix(); bt.nonlinearities(); bt.body_poses(); bt.update_kinematics()
    bt.set_frames([0], np.zeros((1, 3), np.float32)); bt.frame_states(); bt.frame_jacobians()
    bt.set_height_scan([0, 0], np.array([[0.3, 0.0], [0.0, 0.3]], np.float32)); bt.height_scan()
    assert bt.actuator_history().tobytes() == rows.tobytes()
    gc, gv = bt.get_state()
    bt.integrate2()
    e, v = _ev(c, gc, gv, c["pt"])
    _, state = torque(*c["lstm"], e, v, rows, c["tau"][:, d], lim)
    assert _rel(bt.actuator_history(), state) <= REL
    # control_step: one launch, as integrate(SUB)
    a = _setup(capi, monkeypatch, "quadruped_hm", n, seed=62)
    b = _setup(capi, monkeypatch, "quadruped_hm", n, seed=62)
    a["bt"].control_step(a["pt"], SUB, np.empty((n, a["bt"].ob_dim()), np.float32))
    b["bt"].integrate(SUB)
    assert a["bt"].actuator_history().tobytes() == b["bt"].actuator_history().tobytes()
    # force mode: state untouched, tau_ff applied (saturated) on the listed dofs
    bt.set_actuator_history(rows)
    bt.set_control_mode(capi.FORCE_AND_TORQUE)
    bt.integrate(SUB)
    assert bt.actuator_history().tobytes() == rows.tobytes()
    assert np.array_equal(bt.generalized_force()[:, d], np.clip(c["tau"][:, d], -lim, lim))


def test_urdf_and_per_environment_effort_limits_clamp_the_network(capi, monkeypatch):
    n = 256
    c = _setup(capi, monkeypatch, "quadruped_hm", n, seed=71)
    bt, t, d = c["bt"], c["t"], c["dofs"]
    lp, ro = c["lstm"]
    big = (ro[0] * 200.0, ro[1])        # a read-out of hundreds of N m: many dofs reach the URDF limit
    zero = np.zeros((n, len(d), L, 2, HID))
    for rows in (None, "env"):
        elim = _limits(t)[d][None, :]
        if rows is not None:
            ar = np.full((n, t["nv"], 3), -1.0, np.float32)
            elim = np.random.default_rng(7).uniform(2.0, 30.0, (n, 1)).astype(np.float32)
            ar[:, 6:, 2] = elim
            bt.set_actuator_params(ar)
        bt.set_actuator_lstm(d, lp, big)
        gc, gv = bt.get_state()
        bt.integrate(1)
        e, v = _ev(c, gc, gv, c["pt"])
        free = c["tau"][:, d] + net(lp, big, np.stack([e, v], -1), zero)[0]
        got = bt.generalized_force()[:, d]
        lim = np.broadcast_to(elim, free.shape)
        over = np.abs(free) > lim * 1.001
        assert over.mean() > 0.1
        assert np.array_equal(got[over], (np.sign(free) * lim)[over].astype(np.float32))
        assert (np.abs(got) <= lim).all()


def test_an_actuation_delay_feeds_the_delayed_error(capi, monkeypatch):
    """delay 2: after 4 sub-steps of command A, the first sub-step after command B is set still applies A, and the cell sees A's error"""
    n = 128
    c = _setup(capi, monkeypatch, "quadruped_hm", n, seed=73)
    bt, t, d = c["bt"], c["t"], c["dofs"]
    bt.set_actuation_delay(np.full(n, 2, np.int32))
    bt.integrate(SUB)
    ptb = c["pt"].copy(); ptb[:, 7:] += 0.25
    bt.set_pd_target(ptb, np.zeros((n, t["nv"]), np.float32))
    gc, gv = bt.get_state()
    before = bt.actuator_history()
    bt.integrate(1)
    lim = _limits(t)[d]
    ea, v = _ev(c, gc, gv, c["pt"])
    eb, _ = _ev(c, gc, gv, ptb)
    ref_a, st_a = torque(*c["lstm"], ea, v, before, c["tau"][:, d], lim)
    ref_b, _ = torque(*c["lstm"], eb, v, before, c["tau"][:, d], lim)
    got = bt.generalized_force()[:, d]
    assert _rel(got, ref_a) <= REL and _rel(bt.actuator_history(), st_a) <= REL
    assert _rel(got, ref_b) > 1e-2


def test_resets_and_round_trips(capi, monkeypatch):
    import torch
    n = 256
    c = _setup(capi, monkeypatch, "quadruped_hm", n, seed=81)
    bt, d, t = c["bt"], c["dofs"], c["t"]
    zeros = np.zeros((n, len(d), L, 2, HID), np.float32)
    assert bt.actuator_history().tobytes() == zeros.tobytes()          # the set call zeroes
    bt.integrate(SUB)
    assert np.abs(bt.actuator_history()).max() > 0
    bt.set_actuator_lstm(d, *c["lstm"])
    assert bt.actuator_history().tobytes() == zeros.tobytes()
    bt.integrate(SUB)
    bt.set_actuator_history(None, 10, 20)                              # NULL zeroes the range only
    h = bt.actuator_history()
    assert not h[10:30].any() and h[:10].any() and h[30:].any()
    before = bt.actuator_history()
    bt.set_state(c["gc"], c["gv"])                                     # set_state keeps it
    assert bt.actuator_history().tobytes() == before.tobytes()
    # round trips: host, a range, torch _into / _from
    rows = _random_state(np.random.default_rng(3), n, len(d))
    bt.set_actuator_history(rows)
    assert bt.actuator_history().tobytes() == rows.tobytes()
    assert bt.actuator_history(40, 7).tobytes() == rows[40:47].tobytes()
    ht = torch.empty((n, len(d), L, 2, HID), dtype=torch.float32, device="cuda")
    bt.actuator_history_into(ht)
    assert ht.cpu().numpy().tobytes() == rows.tobytes()
    ht[torch.arange(0, n, 3, device="cuda")] = 0.0
    bt.set_actuator_history_from(ht)
    want = rows.copy(); want[::3] = 0.0
    assert bt.actuator_history().tobytes() == want.tobytes()
    bt.set_actuator_history(rows[5:9], 100)
    want[100:104] = rows[5:9]
    assert bt.actuator_history().tobytes() == want.tobytes()
    # non-finite rows are refused, from the host and the device
    for v in (np.nan, np.inf, -np.inf):
        r = rows.copy(); r[n - 1, 3, 1, 1, 7] = v
        with pytest.raises(capi.RsbError, match="not finite"):
            bt.set_actuator_history(r)
        with pytest.raises(capi.RsbError, match="not finite"):
            bt.set_actuator_history_from(torch.from_numpy(r).cuda())
        assert bt.actuator_history().tobytes() == want.tobytes()
    # gym reset zeroes all; a gym-step termination zeroes exactly that environment's rows
    feet = [3, 6]
    bt.gym_configure(c["gc"][0], np.zeros(t["nv"], np.float32), c["pt"][0, 7:], np.full(12, 0.5, np.float32), feet)
    bt.gym_reset()
    assert bt.actuator_history().tobytes() == zeros.tobytes()
    bt.set_state(c["gc"], c["gv"])
    rng = np.random.default_rng(8)
    obs, rew, done = np.empty((n, bt.ob_dim()), np.float32), np.empty(n, np.float32), np.empty(n, np.uint8)
    terminated = 0
    for k in range(30):
        before = bt.actuator_history()
        bt.gym_step(rng.uniform(-3, 3, (n, 12)).astype(np.float32), SUB, obs, rew, done)
        h = bt.actuator_history()
        assert not h[done == 1].any()
        assert (np.abs(h[done == 0]).reshape(int((done == 0).sum()), -1).max(1) > 0).all()
        assert (h[done == 0] != before[done == 0]).any()
        terminated += int(done.sum())
    print(f"{terminated} terminations over 30 gym steps")
    assert terminated > 0


# ---- 4: refusals --------------------------------------------------------------------------------------------------------------------------

def test_refusals_change_nothing(capi, monkeypatch):
    n = 64
    c = _setup(capi, monkeypatch, "quadruped_hm", n, seed=91)
    bt, d = c["bt"], c["dofs"]
    L_ = capi.lib()
    bt.integrate(SUB)
    hist0 = bt.actuator_history()
    params = flat(*c["lstm"])
    P = params.ctypes.data_as(C.c_void_p)

    def call(dl, nd, l=L, h=HID, p=P):
        arr = np.ascontiguousarray(dl, np.int32)
        return L_.rsb_batch_set_actuator_lstm(bt.h, arr.ctypes.data_as(C.c_void_p) if len(arr) else None, nd, l, h, p)
    dofs = np.ascontiguousarray(d, np.int32)
    bad_nan = params.copy(); bad_nan[17] = np.nan
    bad_inf = params.copy(); bad_inf[-1] = np.inf
    for dl, nd in [(dofs, -1), (dofs, 19), (np.r_[dofs[:-1], 18], 12), (np.r_[dofs[:-1], -1], 12), (np.r_[dofs[:-1], 6], 12),
                   (np.r_[dofs[:-1], 3], 12)]:
        assert call(dl, nd) == -1 and L_.rsb_last_error()
        assert bt.actuator_history().tobytes() == hist0.tobytes()
    for kw in (dict(l=0), dict(l=5), dict(h=0), dict(h=33), dict(p=None), dict(p=bad_nan.ctypes.data_as(C.c_void_p)),
               dict(p=bad_inf.ctypes.data_as(C.c_void_p))):
        assert call(dofs, 12, **kw) == -1, kw
        assert bt.actuator_history().tobytes() == hist0.tobytes()
    assert L_.rsb_batch_set_actuator_lstm(bt.h, None, 12, L, HID, P) == -1
    assert b"null dof list" in L_.rsb_last_error()
    rows = np.zeros(hist0.shape, np.float32)
    for eb, ec, wh in ((0, n + 1, capi.HOST), (-1, 2, capi.HOST), (0, 2, 7)):
        assert L_.rsb_batch_set_actuator_history(bt.h, rows.ctypes.data_as(C.c_void_p), eb, ec, wh) == -1
        assert L_.rsb_batch_get_actuator_history(bt.h, rows.ctypes.data_as(C.c_void_p), eb, ec, wh) == -1
    # the same steps as a twin that never saw a refusal
    c2 = _setup(capi, monkeypatch, "quadruped_hm", n, seed=91)
    c2["bt"].integrate(SUB)
    bt.integrate(SUB); c2["bt"].integrate(SUB)
    _same(_outputs(bt), _outputs(c2["bt"]), "after refusals: ")
    assert bt.actuator_history().tobytes() == c2["bt"].actuator_history().tobytes()
    # cleared: the history calls are refused, with the MLP's message
    bt.set_actuator_lstm([], None, None)
    assert L_.rsb_batch_get_actuator_history(bt.h, rows.ctypes.data_as(C.c_void_p), 0, 1, capi.HOST) == -1
    assert b"no actuator network" in L_.rsb_last_error()


# ---- 5: launches, every feature, pybind, the facade ----------------------------------------------------------------------------------

def test_one_launch_per_control_step_and_gym_step(capi, monkeypatch):
    n = 256
    c = _setup(capi, monkeypatch, "quadruped_hm", n, seed=101)
    bt, t = c["bt"], c["t"]
    obs = np.empty((n, bt.ob_dim()), np.float32)
    l0 = bt.launch_count()
    for _ in range(5):
        bt.control_step(c["pt"], SUB, obs)
    assert bt.launch_count() - l0 == 5
    # an LSTM alone (no gains, no rows) lets the gym task run
    b2 = capi.Batch(capi.Model(os.path.join(RSC, "anymal_c_like.urdf")), n)
    b2.set_ground(0.0)
    b2.set_state(c["gc"], c["gv"])
    with pytest.raises(capi.RsbError, match=r"call rsb_batch_set_pd_gains\(\), rsb_batch_set_actuator_params\(\) or rsb_batch_set_actuator_network\(\) first"):
        b2.gym_configure(c["gc"][0], np.zeros(t["nv"], np.float32), c["pt"][0, 7:], np.full(12, 0.5, np.float32), [])
        b2.gym_step(np.zeros((n, 12), np.float32), SUB, obs, np.empty(n, np.float32), np.empty(n, np.uint8))
    b2.set_actuator_lstm(c["dofs"], *c["lstm"])
    rew, done = np.empty(n, np.float32), np.empty(n, np.uint8)
    l0 = b2.launch_count()
    for _ in range(5):
        b2.gym_step(np.zeros((n, 12), np.float32), SUB, obs, rew, done)
    assert b2.launch_count() - l0 == 5
    assert np.isfinite(obs).all()


@pytest.mark.parametrize("name", ["anymal", "atlas"])
def test_every_feature_at_once(capi, monkeypatch, name):
    """inertia, friction and actuator rows, actuation delays, an external wrench, contact bodies, frames, a height scan and IMUs all
    set, with the LSTM on every joint: the first sub-step's torque and rows against the restatement (effort limits from the rows), and
    one launch of SUB equal to SUB launches of one, bit for bit"""
    x = _mix_inputs(name, "DL", 64, seed=43)
    t, n = x["t"], x["n"]
    nb = 6 if t["floating"] else 0
    dofs = np.arange(nb, t["nv"])
    lp, ro = random_lstm(np.random.default_rng(44), L, HID)
    a, b = _mix_batch(capi, monkeypatch, x), _mix_batch(capi, monkeypatch, x)
    for bt in (a, b):
        bt.set_actuator_lstm(dofs, lp, ro)
        bt.set_imus(np.array([0, t["nb"] - 1], np.int32), np.zeros((2, 3), np.float32))
    lim = np.where(x["rows"][:, dofs, 2] >= 0, x["rows"][:, dofs, 2], _limits(t)[dofs][None, :])
    c = dict(t=t, dofs=dofs)
    for k in range(3):
        for bt in (a, b):
            _mix_command(bt, x, k)
        if k == 0:
            _mix_wrench(a, x)
        gc, gv = b.get_state()
        before = b.actuator_history()
        a.integrate(SUB)
        for s in range(SUB):
            if k == 0:
                _mix_wrench(b, x)
            b.integrate(1)
            if k == 0 and s == 0:
                e, v = _ev(c, gc, gv, x["cmds"][0][0])
                ref, st = torque(lp, ro, e, v, before, x["cmds"][0][2][:, dofs], lim)
                assert _rel(b.generalized_force()[:, dofs], ref) <= REL and _rel(b.actuator_history(), st) <= REL
        oa, ob = _outputs(a), _outputs(b)
        oa["hist"], ob["hist"] = a.actuator_history(), b.actuator_history()
        _same(oa, ob, f"{name} control step {k}: ")
        assert not a.diverged().any()


def test_pybind_module(capi, monkeypatch):
    import torch
    from raisimlib_b200 import _rsb_py
    monkeypatch.delenv("RSB_FORCE_WPC", raising=False); monkeypatch.setenv("RSB_FORCE_GENERIC", "0")
    n = 128
    c = _setup(capi, monkeypatch, "quadruped_hm", n, seed=111, network=False)
    path = os.path.join(RSC, "anymal_c_like.urdf")
    pb = _rsb_py.Batch(_rsb_py.Model(path), n, 0)
    with pytest.raises(RuntimeError, match="set_actuator_lstm: 3 parameters"):
        pb.set_actuator_lstm([6, 7], L, HID, [0.0, 1.0, 2.0])
    params = flat(*c["lstm"])
    assert len(params) == count(L, HID)
    pb.set_actuator_lstm([int(i) for i in c["dofs"]], L, HID, params.tolist())
    rows = torch.from_numpy(_random_state(np.random.default_rng(4), n, 12)).cuda()
    pb.set_actuator_history(rows.data_ptr(), 0, n)
    back = torch.zeros_like(rows)
    pb.actuator_history(back.data_ptr(), 0, n); pb.sync()
    assert torch.equal(back, rows)
    pb.set_actuator_lstm([], 0, 0, [])
    with pytest.raises(RuntimeError, match="no actuator network"):
        pb.actuator_history(back.data_ptr(), 0, n)


def test_cpp_actuator_lstm_example():
    """the facade example (examples/actuator_lstm.cpp): one launch per control step, resets through resetActuatorHistory, and a batch
    of 256 against stand-alone Worlds bit for bit"""
    exe = os.path.join(ROOT, "examples", "actuator_lstm")
    if not os.path.exists(exe):
        subprocess.check_call(["make", "-C", os.path.join(ROOT, "examples")])
    out = subprocess.run([exe, os.path.join(RSC, "anymal_c_like.urdf")], capture_output=True, text=True, timeout=600)
    print(out.stdout)
    assert out.returncode == 0, out.stdout + out.stderr
    assert "launches per control step 1.00" in out.stdout and ", 0 differ" in out.stdout
