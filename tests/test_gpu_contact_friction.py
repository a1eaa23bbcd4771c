"""Per-environment terrain friction (rsb_batch_set_contact_friction / rsb_batch_clear_contact_friction) through the C-ABI on an H100
(pytest -m gpu): bit-identity with the batch-level friction on every compiled instance, every environment against a float64 oracle
configured with that environment's frictions, a box on a slope, isolation and persistence, launch shapes, and the rules of the
contract (sources, refusals, launch count, the C++ facade)."""
import ctypes as C
import os
import subprocess

import numpy as np
import pytest

from conftest import ROOT, RSC
from helpers import ANYMAL_GC0, BOX_URDF, THRESH, setup_batch
from oracle.oracle import Oracle
from test_gpu_contact_forces import _make, _outputs, _same
from test_self_collision_oracle import anymal_leg_pairs, crossed_anymal

pytestmark = pytest.mark.gpu

SUB = 4
FOOT_MU = (0.3, 0.5, 0.7, 1.1)       # batch-level friction of the feet (rsb_batch_set_collision_friction) where a case sets it


@pytest.fixture(scope="module")
def capi():
    import torch
    assert torch.cuda.is_available(), "GPU tests need a CUDA device"
    from raisimlib_b200 import capi as c
    return c


def _feet(t):
    return [i for i, nme in enumerate(t["coll_names"]) if nme.endswith("_FOOT")]


# name -> (case of test_gpu_contact_forces, terrain, self-collision pairs)
SETUPS = {"quadruped_hm": ("quadruped", "hm", False), "humanoid_ground": ("humanoid", "ground", False), "generic_self": ("generic", "hm", True)}


def _setup(capi, monkeypatch, which, n, seed, wpc=None):
    """_make's robots; the feet (where the model has them) on batch-level frictions; the leg pairs on the generic instance"""
    case, terrain, pairs = SETUPS[which]
    c = _make(capi, monkeypatch, case, n, terrain, seed, wpc=wpc, oracles=False)
    for k, ci in enumerate(_feet(c["t"])):
        c["bt"].set_collision_friction(ci, FOOT_MU[k % 4])
    if pairs:
        c["bt"].set_self_collision(anymal_leg_pairs())
    return c


def _random_rows(t, n, seed):
    """a different row in every environment: mu in [0, 1.5], some exact 0 and some -1"""
    rng = np.random.default_rng(seed)
    rows = rng.uniform(0.0, 1.5, (n, t["ncoll"]))
    rows[rng.random((n, t["ncoll"])) < 0.1] = 0.0
    rows[rng.random((n, t["ncoll"])) < 0.15] = -1.0
    return rows.astype(np.float32)


def _batch_values(c):
    """the row every environment resolves to without rows: the feet's batch-level friction, params mu elsewhere"""
    t, bt = c["t"], c["bt"]
    row = np.full(t["ncoll"], bt.get_params().mu, np.float32)
    for k, ci in enumerate(_feet(t)):
        row[ci] = FOOT_MU[k % 4]
    return np.tile(row, (c["n"], 1))


def _all_outputs(bt):
    o = _outputs(bt)
    f, s = bt.body_contact_forces()
    o.update(f=f, s=s)
    return o


# ---- 1: bit-identity with the batch-level friction -------------------------------------------------------------------------------------

@pytest.mark.parametrize("which", list(SETUPS))
def test_no_rows_minus_one_reset_cleared_and_batch_values_agree(capi, monkeypatch, which):
    """no rows, rows of -1, rows reset with NULL, rows set then cleared, and rows equal to the batch-level values: every output of 8
    control steps bit for bit, including the per-body contact forces"""
    n = 300
    runs = {}
    for mode in ("never", "minus_one", "null_reset", "cleared", "batch_values"):
        c = _setup(capi, monkeypatch, which, n, seed=61)
        bt = c["bt"]
        bt.set_contact_bodies(list(range(min(c["t"]["nb"], 32))))
        if mode == "minus_one":
            bt.set_contact_friction(np.full((n, c["t"]["ncoll"]), -1.0, np.float32))
        elif mode == "null_reset":
            bt.set_contact_friction(_random_rows(c["t"], n, 3))
            bt.set_contact_friction(None)
        elif mode == "cleared":
            bt.set_contact_friction(_random_rows(c["t"], n, 3))
            bt.integrate(SUB); bt.set_state(c["gc"], c["gv"])
            bt.clear_contact_friction()
        elif mode == "batch_values":
            bt.set_contact_friction(_batch_values(c))
        runs[mode] = []
        for k in range(8):
            bt.integrate(SUB)
            runs[mode].append(_all_outputs(bt))
    assert runs["never"][-1]["cnt"].sum() > n
    for mode in runs:
        for k in range(8):
            _same(runs["never"][k], runs[mode][k], f"{which} {mode}, control step {k}: ")


# ---- 2: against the oracle -----------------------------------------------------------------------------------------------------------

def test_every_environment_matches_an_oracle_with_its_frictions(capi):
    """256 quadrupeds, every one with its own row (mu in [0, 1.5], some exact 0, some -1 on top of a batch-level foot friction),
    against a float64 oracle per environment configured through set_collision_friction: the bounds of
    test_per_body_friction_matches_oracle"""
    n = 256
    t, bt, o64, _, gc, gv, tau = setup_batch(capi, "anymal_c_like.urdf", n, seed=171, base_z=0.55, joint_scale=0.2, vel=1.0)
    foot = _feet(t)[0]
    bt.set_collision_friction(foot, 0.35)
    rows = _random_rows(t, n, 5)
    bt.set_contact_friction(rows)
    bt.integrate(20)
    g, _ = bt.get_state()
    a, b = gc.copy(), gv.copy()
    mu_default = bt.get_params().mu
    for e in range(n):
        o = Oracle(t, params=dict(threshold=THRESH))
        o.set_ground(0.0)
        for ci in range(t["ncoll"]):
            r = float(rows[e, ci])
            o.set_collision_friction(ci, r if r >= 0 else (0.35 if ci == foot else mu_default))
        ae, be = a[e:e + 1].copy(), b[e:e + 1].copy()
        o.step(ae, be, n_steps=20, tau_ff=tau[e:e + 1])
        a[e], b[e] = ae[0], be[0]
    err = np.abs(g - a).max(1)
    print(f"per-environment friction 20-step error median {np.median(err):.2e} p90 {np.quantile(err, 0.9):.2e}")
    assert np.median(err) < 2e-5 and np.quantile(err, 0.9) < 2e-3
    # the rows matter: in the environments whose feet or legs slide, the batch-level oracle ends millimetres or more away
    a0, b0 = gc.copy(), gv.copy()
    o64.set_collision_friction(foot, 0.35)
    o64.step(a0, b0, n_steps=20, tau_ff=tau)
    assert (np.abs(g - a0).max(1) > 1e-3).sum() > n // 4


# ---- 3: physics ---------------------------------------------------------------------------------------------------------------------

def test_box_on_a_slope_slides_or_sticks_by_its_friction(capi):
    """a box on a 20 degree slope (tilted gravity) in 64 environments with mu from 0 to 0.7: below tan 20 it slides with acceleration
    g (sin - mu cos) within 0.03 m/s^2 (the float64 oracle is within 0.015 up to mu = 0.35), above it sticks, and mu = 0 gives no
    tangential impulse"""
    n, th, g, dt = 64, np.deg2rad(20.0), 9.81, 0.0025
    bt = capi.Batch(capi.Model(BOX_URDF), n)
    bt.set_ground(0.0)
    bt.set_params(threshold=THRESH, gravity=(g * np.sin(th), 0.0, -g * np.cos(th)))
    mu = np.linspace(0.0, 0.7, n).astype(np.float32)
    bt.set_contact_friction(mu[:, None])
    gc = np.zeros((n, 7), np.float32); gc[:, 1] = np.arange(n); gc[:, 2] = 0.0999; gc[:, 3] = 1.0
    bt.set_state(gc, np.zeros((n, 6), np.float32))
    bt.integrate(40)
    v40 = bt.get_state()[1][:, 0].astype(np.float64)
    bt.integrate(60)
    gN, vN = bt.get_state()
    ct, cnt = bt.contacts()
    acc = (vN[:, 0] - v40) / (60 * dt)
    expected = np.maximum(g * (np.sin(th) - mu * np.cos(th)), 0.0)
    assert np.isfinite(gN).all() and np.isfinite(vN).all() and np.isfinite(ct["impulse"]).all()
    slide, stick = mu < 0.33, mu > 0.40
    print(f"slope: |a - g(sin - mu cos)| max {np.abs(acc - expected)[slide].max():.4f} m/s^2; sticking |v| max {np.abs(vN[stick]).max():.1e}")
    assert np.abs(acc - expected)[slide].max() < 0.03
    assert np.abs(vN[stick]).max() < 1e-4
    assert (cnt > 0).all()
    live = np.arange(ct.shape[1])[None] < cnt[:, None]
    tangential = np.abs(ct["impulse"][0, :, :2])[live[0]]
    assert tangential.max() <= 1e-7 * ct["impulse"][0, :, 2].max(), tangential


# ---- 4: isolation and persistence ----------------------------------------------------------------------------------------------------

def test_a_range_leaves_every_other_environment_alone(capi, monkeypatch):
    n, lo, hi = 300, 100, 200
    out = {}
    for mode in ("never", "range"):
        c = _setup(capi, monkeypatch, "quadruped_hm", n, seed=63)
        if mode == "range":
            c["bt"].set_contact_friction(np.full((hi - lo, c["t"]["ncoll"]), 0.05, np.float32), env_begin=lo)
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
        c = _setup(capi, monkeypatch, "generic_self", n, seed=65)
        bt, t = c["bt"], c["t"]
        rows = _random_rows(t, n, 9)
        if mode == "before":
            bt.set_contact_friction(rows)
        bt.set_collision_friction(_feet(t)[1], 0.9)
        bt.set_self_collision(anymal_leg_pairs()[:6])
        H = (0.1 * np.random.default_rng(65).uniform(-1, 1, (49, 65))).astype(np.float32)
        bt.clear_terrain()
        bt.set_heightmap(65, 49, 12.8, 9.6, 0.1, -0.2, H)
        bt.set_params(mu=0.6)
        if mode == "after":
            bt.set_contact_friction(rows)
        for k in range(4):
            bt.integrate(SUB)
        out[mode] = _outputs(bt)
    _same(out["after"], out["before"], "rows set before the rebuilds: ")
    assert out["after"]["gc"].tobytes() != out["none"]["gc"].tobytes()


def test_gym_resets_keep_the_rows(capi, monkeypatch):
    """the gym task's steps and resets leave the rows in place: from the state they leave, the batch steps as a fresh batch with the
    same rows does, and unlike one without them"""
    n = 256
    g = _setup(capi, monkeypatch, "quadruped_hm", n, seed=67)
    rows = np.full((n, g["t"]["ncoll"]), 0.05, np.float32)
    g["bt"].set_contact_friction(rows)
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
            b = _setup(capi, monkeypatch, "quadruped_hm", n, seed=67)["bt"]
            if mode == "same":
                b.set_contact_friction(rows)
        b.set_state(gc, gv); b.set_pd_target(gc, np.zeros((n, 18), np.float32))
        for k in range(3):
            b.integrate(SUB)
        res[mode] = b.get_state()[0]
    assert res["gym"].tobytes() == res["same"].tobytes()
    assert res["gym"].tobytes() != res["none"].tobytes()


def test_self_contacts_keep_their_pair_friction(capi, monkeypatch):
    """crossed legs in the air: only self contacts, so any friction rows change nothing, bit for bit"""
    n = 256
    out = {}
    for mode in ("none", "rows"):
        c = _make(capi, monkeypatch, "generic", n, "ground", seed=69, oracles=False)
        bt, t = c["bt"], c["t"]
        bt.set_self_collision(anymal_leg_pairs(), mu=0.4)
        gc = crossed_anymal(n, np.random.default_rng(69)).astype(np.float32)
        bt.set_state(gc, np.zeros((n, t["nv"]), np.float32)); bt.set_pd_target(gc, np.zeros((n, t["nv"]), np.float32))
        if mode == "rows":
            bt.set_contact_friction(np.zeros((n, t["ncoll"]), np.float32))
        bt.integrate(SUB)
        out[mode] = _outputs(bt)
    pts, cnt = out["none"]["pts"], out["none"]["cnt"]
    live = np.arange(pts.shape[1])[None] < cnt[:, None]
    assert cnt.sum() > n and (pts[live] >= c["t"]["npts"]).all(), "expected self contacts only"
    _same(out["none"], out["rows"], "self contacts with friction rows: ")


# ---- 5: launch shapes -----------------------------------------------------------------------------------------------------------------

@pytest.mark.parametrize("which", list(SETUPS))
def test_every_launch_shape_gives_the_same_results(capi, monkeypatch, which):
    """a distinct row in every environment: every CTA size that fits, the sub-step barrier and the paired stage A on and off, a
    partly filled last round -- the same results bit for bit"""
    n = 2300 if which.startswith("humanoid") else 4500
    ref, taken = None, []
    shapes = [(None, "1", "1")] + [(w, "1", "1") for w in (28, 16, 14, 8, 4, 1)] + [(None, "0", "1"), (None, "1", "0")]
    for wpc, barrier, pair in shapes:
        monkeypatch.setenv("RSB_SUBSTEP_BARRIER", barrier); monkeypatch.setenv("RSB_PAIR_STAGE_A", pair)
        c = _setup(capi, monkeypatch, which, n, seed=71, wpc=wpc)
        if wpc is not None and c["cfg"]["wpc"] != wpc:
            continue                                                          # did not fit
        taken.append(c["cfg"]["wpc"])
        c["bt"].set_contact_friction(_random_rows(c["t"], n, 7))
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


# ---- 6: the interface -------------------------------------------------------------------------------------------------------------------

def test_pinned_pageable_device_and_pybind_sources_agree(capi, monkeypatch):
    import torch
    from raisimlib_b200 import _rsb_py
    n = 200
    out = {}
    for mode in ("pageable", "pinned", "device", "raw", "pybind"):
        c = _setup(capi, monkeypatch, "quadruped_hm", n, seed=73)
        bt = c["bt"]
        rows = _random_rows(c["t"], n, 11)
        if mode == "pageable":
            bt.set_contact_friction(rows[50:], env_begin=50); bt.set_contact_friction(rows[:50])
        elif mode == "pinned":
            p = torch.from_numpy(rows).pin_memory()
            assert capi.lib().rsb_batch_set_contact_friction(bt.h, C.c_void_p(p.data_ptr()), 0, n, capi.HOST) == 0
        elif mode == "device":
            bt.set_contact_friction_from(torch.from_numpy(rows).cuda())
        elif mode == "raw":
            tr = torch.from_numpy(rows).cuda()
            assert capi.lib().rsb_batch_set_contact_friction(bt.h, C.c_void_p(tr.data_ptr()), 0, n, capi.DEVICE) == 0
        for k in range(3):
            bt.integrate(SUB)
        out[mode] = _outputs(bt)
    for mode in ("pinned", "device", "raw"):
        _same(out["pageable"], out[mode], f"{mode} source: ")
    c = _setup(capi, monkeypatch, "quadruped_hm", n, seed=73)
    with pytest.raises(ValueError):
        c["bt"].set_contact_friction_from(torch.from_numpy(rows).double().cuda())
    with pytest.raises(ValueError):
        c["bt"].set_contact_friction_from(torch.from_numpy(rows[:, :-1].copy()).cuda())
    with pytest.raises(ValueError):
        c["bt"].set_contact_friction_from(torch.from_numpy(np.ascontiguousarray(rows[:, :8].T)).cuda().T)
    with pytest.raises(ValueError):
        c["bt"].set_contact_friction_from(torch.from_numpy(rows))
    with pytest.raises(ValueError):
        c["bt"].set_contact_friction(rows[:, :-1])
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
    tr = torch.from_numpy(rows).cuda()
    torch.cuda.synchronize()
    pb.set_contact_friction(tr.data_ptr(), 0, n); bt.set_contact_friction(rows)
    pb.integrate(SUB); bt.integrate(SUB); pb.sync()
    assert torch.from_dlpack(pb.gc()).cpu().numpy().tobytes() == bt.get_state()[0].tobytes()


def test_refusals_change_nothing(capi, monkeypatch):
    import torch
    n = 200
    L = capi.lib()
    assert L.rsb_batch_set_contact_friction(None, None, 0, 1, capi.HOST) == -1
    assert L.rsb_batch_clear_contact_friction(None) == -1
    runs = {}
    for mode in ("clean", "refused", "first_refused", "never"):
        c = _setup(capi, monkeypatch, "quadruped_hm", n, seed=75)
        bt, ncoll = c["bt"], c["t"]["ncoll"]
        rows = _random_rows(c["t"], n, 13)
        if mode == "clean":
            bt.set_contact_friction(rows)
        if mode in ("refused", "first_refused"):
            if mode == "refused":
                bt.set_contact_friction(rows)
            for v in (np.nan, np.inf, -np.inf):
                for e, ci in ((0, 0), (57, ncoll // 2), (n - 1, ncoll - 1)):
                    r = rows.copy(); r[e, ci] = v
                    for where in (capi.HOST, capi.DEVICE):
                        src = torch.from_numpy(r).cuda() if where == capi.DEVICE else r
                        ptr = C.c_void_p(src.data_ptr()) if where == capi.DEVICE else r.ctypes.data_as(C.c_void_p)
                        assert L.rsb_batch_set_contact_friction(bt.h, ptr, 0, n, where) == -1, (v, e, ci)
                        assert b"no row changed" in L.rsb_last_error()
                        assert f"environment {e}, collision body {ci}".encode() in L.rsb_last_error()
            ok = rows.ctypes.data_as(C.c_void_p)
            for begin, count, where in ((n - 1, 2, capi.HOST), (-1, 1, capi.HOST), (0, -1, capi.HOST), (0, n, 2), (0, n, -1)):
                assert L.rsb_batch_set_contact_friction(bt.h, ok, begin, count, where) == -1, (begin, count, where)
            assert L.rsb_batch_set_contact_friction(bt.h, None, 0, n + 1, capi.HOST) == -1
        runs[mode] = []
        for k in range(3):
            bt.integrate(SUB)
            runs[mode].append(_outputs(bt))
    for k in range(3):
        _same(runs["clean"][k], runs["refused"][k], f"after refusals, step {k}: ")
        _same(runs["never"][k], runs["first_refused"][k], f"refused first call, step {k}: ")


def test_rows_add_no_launch(capi, monkeypatch):
    """setting, resetting and clearing rows launches nothing the batch counts, and a step with rows is one launch"""
    n = 128
    c = _setup(capi, monkeypatch, "quadruped_hm", n, seed=77)
    bt = c["bt"]
    bt.mass_matrix()                                  # the getters' buffers are fresh: rows must not make them stale
    L0 = bt.launch_count()
    bt.set_contact_friction(_random_rows(c["t"], n, 15))
    bt.set_contact_friction(None, env_begin=10, env_count=5)
    bt.mass_matrix()
    assert bt.launch_count() == L0
    bt.integrate(SUB)
    assert bt.launch_count() == L0 + 1
    bt.clear_contact_friction()
    bt.integrate(SUB)
    assert bt.launch_count() == L0 + 2


def test_cpp_friction_randomization_example():
    """the raisim:: facade: setMaterialPairProp in an upstream-shaped reset(), one launch per control step, every environment equal to
    a stand-alone World with the same frictions (examples/friction_randomization.cpp)"""
    exe = os.path.join(ROOT, "examples", "friction_randomization")
    if not os.path.exists(exe):
        subprocess.check_call(["make", "-C", os.path.join(ROOT, "examples")])
    out = subprocess.run([exe, os.path.join(RSC, "anymal_c_like.urdf")], capture_output=True, text=True, timeout=600)
    print(out.stdout)
    assert out.returncode == 0, out.stdout + out.stderr
