"""Per-environment inertial parameters (rsb_batch_set_body_inertia / rsb_batch_clear_body_inertia) through the C-ABI on an H100
(pytest -m gpu): every compiled instance against one float64 and one float32 oracle per parameter set, known answers, bit-identity
with the model's values and across launch shapes, and the rules of the contract (laziness, sources, refusals, gym resets, devices)."""
import ctypes as C
import os
import subprocess

import numpy as np
import pytest

from body_inertia_ref import add_payload, randomized, rows_of, tables_with
from conftest import ROOT, RSC
from helpers import ANYMAL_GC0, SPHERE_URDF, THRESH, index_parity, launch_config
from oracle.oracle import Oracle
from oracle.urdf_tables import load_tables
from test_gpu_contact_forces import CASES, _make, _outputs, _same

pytestmark = pytest.mark.gpu

SUB, DT, G = 4, 0.0025, 9.81
GROUPS = 16


@pytest.fixture(scope="module")
def capi():
    import torch
    assert torch.cuda.is_available(), "GPU tests need a CUDA device"
    from raisimlib_b200 import capi as c
    return c


def _sets(t, seed):
    rng = np.random.default_rng(seed)
    return [randomized(t, rng) for _ in range(GROUPS)]


def _rows(sets, n):
    """environment e takes parameter set e % GROUPS: neighbours, and the partners of the paired stage A (e, e + 4), differ"""
    return np.stack([rows_of(*sets[e % GROUPS]) for e in range(n)])


def _distinct_rows(t, n, seed):
    """a different row in every environment"""
    rng = np.random.default_rng(seed)
    nb = t["nb"]
    mass = t["mass"][None] * rng.uniform(0.7, 1.3, (n, nb))
    com = t["com"][None] + rng.uniform(-0.02, 0.02, (n, nb, 3))
    inertia = t["inertia"][None] * rng.uniform(0.7, 1.3, (n, nb, 1))
    return np.concatenate([mass[:, :, None], com, inertia], axis=2).astype(np.float32)


def _oracles(t, sets, terrain, seed):
    """[float64, float32] oracle per parameter set, on the terrain _make built"""
    H = None if terrain == "ground" else (0.1 * np.random.default_rng(seed).uniform(-1, 1, (49, 65))).astype(np.float32).astype(np.float64)
    out = []
    for mass, com, inertia in sets:
        u = tables_with(t, mass, com, inertia)
        pair = [Oracle(u, params=dict(threshold=THRESH)), Oracle(u, precision="f32", params=dict(threshold=THRESH))]
        for o in pair:
            if H is None:
                o.set_ground(0.0)
            else:
                o.set_heightmap(65, 49, 12.8, 9.6, 0.1, -0.2, H)
        out.append(pair)
    return out


def _step_groups(ors, which, c, gc, gv, n_steps, debug=False):
    """step every group of environments on its own oracle (which: 0 float64, 1 float32); gc / gv updated in place, debug outputs merged"""
    n, nv = gc.shape[0], gv.shape[1]
    merged = {}
    for g in range(GROUPS):
        idx = np.arange(g, n, GROUPS)
        a, b = gc[idx], gv[idx]
        d = ors[g][which].step(a, b, n_steps=n_steps, ptarget=c["pt"][idx].astype(np.float64), vtarget=np.zeros((len(idx), nv)), kp=c["kp"], kd=c["kd"], debug=debug)
        gc[idx], gv[idx] = a, b
        for k, v in (d or {}).items():
            merged.setdefault(k, np.zeros((n,) + v.shape[1:], v.dtype))[idx] = v
    return merged


def _all_outputs(bt):
    """_outputs plus M, h, poses and the per-body contact forces"""
    o = _outputs(bt)
    R, p = bt.body_poses()
    f, s = bt.body_contact_forces()
    o.update(M=bt.mass_matrix(), h=bt.nonlinearities(), R=R, p=p, f=f, s=s)
    return o


# ---- 1: against the oracle ---------------------------------------------------------------------------------------------------------

@pytest.mark.parametrize("terrain", ["ground", "hm"])
@pytest.mark.parametrize("name", list(CASES))
def test_parity_with_one_oracle_per_parameter_set(capi, monkeypatch, name, terrain):
    """512 environments in 16 parameter sets (masses x U(0.7, 1.3), centres of mass moved up to 2 cm, inertias rescaled and turned),
    stiff PD: M and h of the getters, the contact lists of one step (bit-exact outside the margin), the state after 1 and 10 steps,
    at the bounds of tests/test_gpu_instances.py"""
    n = 512
    seed = 900 + 7 * len(name) + (terrain == "hm")
    c = _make(capi, monkeypatch, name, n, terrain, seed, oracles=False)
    bt, t = c["bt"], c["t"]
    sets = _sets(t, seed)
    bt.set_body_inertia(_rows(sets, n))
    ors = _oracles(t, sets, terrain, seed)
    gc, gv = c["gc"].astype(np.float64), c["gv"].astype(np.float64)
    M, h = bt.mass_matrix(), bt.nonlinearities()
    a, b = gc.copy(), gv.copy()
    d = _step_groups(ors, 0, c, a, b, 1, debug=True)
    Ms, hs = np.abs(d["M"]).max(), np.abs(d["h"]).max()
    eM, eh = np.abs(M - d["M"]).max(), np.abs(h - d["h"]).max()
    print(f"{name} {terrain}: M {eM:.2e}/{Ms:.1e}  h {eh:.2e}/{hs:.1e}")
    assert eM < 2e-6 * Ms and eh < 2e-6 * max(hs, 1.0) * 10
    # the parameters matter: the model's M is far from these
    d0 = Oracle(t).step(gc.copy(), gv.copy(), debug=True)
    assert np.abs(d0["M"] - d["M"]).max() > 100 * eM
    bt.integrate(1)
    g1, v1 = bt.get_state(); ct, cnt = bt.contacts(); pts = bt.contact_points(); st = bt.solver_status()
    c_, e_ = gc.copy(), gv.copy()
    d32 = _step_groups(ors, 1, c, c_, e_, 1, debug=True)
    assert np.isfinite(g1).all() and cnt.sum() > n // 4
    hard = index_parity(pts, cnt, d32, f"{name} {terrain}")
    assert hard.sum() <= (0 if terrain == "ground" else 1), f"contact lists differ in envs {np.where(hard)[0][:10]}"
    same = (pts == d["c_pt"]).all(1)
    conv = same & (st == 0) & (d["status"] == 0)
    ev = np.abs(v1 - b)[conv]; eq = np.abs(g1 - a)[conv]; e32 = np.abs(e_ - b)[conv]
    scale_v = 1.0 + np.abs(b[conv])
    assert conv.mean() > 0.88
    assert np.median(ev.max(1)) < max(2e-5, 3 * np.median(e32.max(1)))
    assert np.max(ev / scale_v) < max(5e-3, 3 * np.max(e32 / scale_v))
    assert eq.max() < 5e-3 * DT * (1.0 + np.abs(b[conv]).max()) + 2e-6
    bt.integrate(9)
    gN, _ = bt.get_state()
    _step_groups(ors, 0, c, a, b, 9)
    _step_groups(ors, 1, c, c_, e_, 9)
    e = np.abs(gN - a).max(1); ef = np.abs(c_ - a).max(1)
    print(f"   10 steps: gc err median {np.median(e):.1e} p90 {np.quantile(e, .9):.1e} p99 {np.quantile(e, .99):.1e} (f32 oracle p99 {np.quantile(ef, .99):.1e})")
    assert np.isfinite(gN).all()
    assert np.median(e) < 2e-5 and np.median(e) < 5 * np.median(ef) + 1e-6
    assert np.quantile(e, 0.9) < max(1e-4, 5 * np.quantile(ef, 0.9))
    assert np.quantile(e, 0.99) < max(5e-3, 5 * np.quantile(ef, 0.99))


# ---- 2: known answers ----------------------------------------------------------------------------------------------------------------

def test_resting_spheres_carry_their_own_weight(capi):
    """a sphere resting on the plane in every environment, each with its own mass: normal impulse m_e g dt"""
    n = 64
    t = load_tables(SPHERE_URDF)
    bt = capi.Batch(capi.Model(SPHERE_URDF), n)
    bt.set_ground(0.0)
    m = np.random.default_rng(2).uniform(0.2, 20.0, n)
    rows = np.tile(bt.model_body_inertia(), (n, 1, 1))
    rows[:, 0, 0] = m; rows[:, 0, 4:] = t["inertia"][0] * (m / t["mass"][0])[:, None]
    bt.set_body_inertia(rows)
    gc = np.zeros((n, 7), np.float32); gc[:, 0] = np.arange(n); gc[:, 2] = 0.0999; gc[:, 3] = 1.0
    bt.set_state(gc, np.zeros((n, 6), np.float32))
    bt.integrate(1)
    ct, cnt = bt.contacts()
    assert (cnt == 1).all()
    mg = rows[:, 0, 0].astype(np.float64) * G * DT
    assert np.abs(ct["impulse"][:, 0, 2] - mg).max() < 1e-4 * mg.max()
    assert np.abs(ct["impulse"][:, 0, 2] / mg - 1).max() < 1e-4


def test_standing_robots_with_payloads_carry_robot_and_payload(capi, monkeypatch):
    """ANYmal-like robots standing with a base payload of 0-10 kg each (mass and centre of mass offset composed onto the base): after
    2 s the feet carry (m_robot + m_payload,e) g within 2 %"""
    monkeypatch.delenv("RSB_FORCE_WPC", raising=False); monkeypatch.setenv("RSB_FORCE_GENERIC", "0")
    path = os.path.join(RSC, "anymal_c_like.urdf")
    t = load_tables(path)
    n = 64
    bt = capi.Batch(capi.Model(path), n)
    bt.set_ground(0.0)
    rng = np.random.default_rng(6)
    payload = np.linspace(0.0, 10.0, n)
    rows = np.tile(bt.model_body_inertia(), (n, 1, 1))
    for e in range(n):
        pos = np.r_[rng.uniform(-0.05, 0.05, 2), rng.uniform(0.05, 0.1)]
        m, c_, I = add_payload(t["mass"][0], t["com"][0], t["inertia"][0], payload[e], pos, (0.02, 0, 0, 0.02, 0, 0.03))
        rows[e, 0] = np.r_[m, c_, I]
    bt.set_body_inertia(rows)
    gc = np.tile(ANYMAL_GC0.astype(np.float32), (n, 1)); gc[:, 2] = 0.54
    gc[:, 7:] += rng.uniform(-0.05, 0.05, (n, 12)).astype(np.float32)
    kp = np.r_[np.zeros(6), 300.0 * np.ones(12)]; kd = np.r_[np.zeros(6), 8.0 * np.ones(12)]
    bt.set_control_mode(capi.PD_PLUS_FEEDFORWARD_TORQUE); bt.set_pd_gains(kp, kd)
    bt.set_pd_target(gc, np.zeros((n, 18), np.float32)); bt.set_state(gc, np.zeros((n, 18), np.float32))
    bt.set_contact_bodies_by_name(["LF_FOOT", "RF_FOOT", "LH_FOOT", "RH_FOOT"])
    for k in range(200):
        bt.integrate(SUB)
    f, s = bt.body_contact_forces()
    weight = (t["mass"].sum() + payload) * G
    assert (s == SUB).all()
    err = np.abs(f[:, :, 2].sum(1) - weight) / weight
    print(f"feet carry the weight within {100 * err.max():.3f} %")
    assert err.max() < 0.02


# ---- 3: bit-identity -------------------------------------------------------------------------------------------------------------------

@pytest.mark.parametrize("name", list(CASES))
def test_model_rows_and_cleared_rows_change_nothing(capi, monkeypatch, name):
    """rows equal to the model's values, and rows set then cleared, give every output of a batch that never set any, bit for bit, over
    10 control steps"""
    runs = {}
    for mode in ("never", "model", "cleared"):
        c = _make(capi, monkeypatch, name, 300, "hm", seed=41, oracles=False)
        bt = c["bt"]
        bt.set_contact_bodies(list(range(min(c["t"]["nb"], 32))))
        if mode == "model":
            bt.set_body_inertia(np.tile(bt.model_body_inertia(), (300, 1, 1)))
        if mode == "cleared":
            bt.set_body_inertia(_distinct_rows(c["t"], 300, 3))
            bt.integrate(SUB); bt.set_state(c["gc"], c["gv"])
            bt.clear_body_inertia()
        runs[mode] = []
        for k in range(10):
            bt.integrate(SUB)
            runs[mode].append(_all_outputs(bt))
    for mode in ("model", "cleared"):
        for k in range(10):
            _same(runs["never"][k], runs[mode][k], f"{name} {mode}, control step {k}: ")


def test_a_range_leaves_every_other_environment_alone(capi, monkeypatch):
    n, lo, hi = 300, 100, 200
    out = {}
    for mode in ("never", "range"):
        c = _make(capi, monkeypatch, "quadruped", n, "hm", seed=43, oracles=False)
        if mode == "range":
            c["bt"].set_body_inertia(_distinct_rows(c["t"], hi - lo, 5), env_begin=lo)
        for k in range(5):
            c["bt"].integrate(SUB)
        out[mode] = _outputs(c["bt"])
        out[mode].update(M=c["bt"].mass_matrix())
    keep = np.r_[0:lo, hi:n]
    for k in out["never"]:
        a, b = np.asarray(out["never"][k]), np.asarray(out["range"][k])
        assert a[keep].tobytes() == b[keep].tobytes(), f"{k} differs outside the range"
    assert (out["never"]["gc"][lo:hi] != out["range"]["gc"][lo:hi]).any(1).all()


@pytest.mark.parametrize("name", list(CASES))
def test_every_launch_shape_gives_the_same_results(capi, monkeypatch, name):
    """a distinct row in every environment: every CTA size that fits, the sub-step barrier and the paired stage A on and off, a
    partly filled last round -- the same results bit for bit (a leader reading its own row for its partner would show here)"""
    n = 2300 if name == "humanoid" else 4500
    ref, taken = None, []
    shapes = [(None, "1", "1")] + [(w, "1", "1") for w in (28, 16, 14, 8, 4, 1)] + [(None, "0", "1"), (None, "1", "0")]
    for wpc, barrier, pair in shapes:
        monkeypatch.setenv("RSB_SUBSTEP_BARRIER", barrier); monkeypatch.setenv("RSB_PAIR_STAGE_A", pair)
        c = _make(capi, monkeypatch, name, n, "hm", seed=47, wpc=wpc, oracles=False)
        if wpc is not None and c["cfg"]["wpc"] != wpc:
            continue                                                          # did not fit
        taken.append(c["cfg"]["wpc"])
        c["bt"].set_body_inertia(_distinct_rows(c["t"], n, 7))
        for k in range(2):
            c["bt"].integrate(SUB)
        g, v = c["bt"].get_state()
        ct, cnt = c["bt"].contacts()
        res = (g.tobytes(), v.tobytes(), ct.tobytes(), cnt.tobytes(), c["bt"].mass_matrix().tobytes())
        if ref is None:
            ref = res
            T = c["cfg"]["wpc"] * c["cfg"]["grid"]
            assert n % T != 0 and cnt.any()
        assert res == ref, f"{name}: differs at wpc {wpc} barrier {barrier} pairing {pair}"
        del c
    assert len(set(taken)) >= 5


# ---- 4: the interface ------------------------------------------------------------------------------------------------------------------

def test_getters_see_new_rows_at_the_cost_of_one_kinematics_pass(capi, monkeypatch):
    n = 128
    c = _make(capi, monkeypatch, "quadruped", n, "ground", seed=51, oracles=False)
    bt, t = c["bt"], c["t"]
    M0 = bt.mass_matrix()
    L0 = bt.launch_count()
    sets = _sets(t, 51)
    bt.set_body_inertia(_rows(sets, n))
    M1 = bt.mass_matrix()
    assert bt.launch_count() == L0 + 1
    h1 = bt.nonlinearities(); bt.body_poses()
    assert bt.launch_count() == L0 + 1
    d = _step_groups(_oracles(t, sets, "ground", 51), 0, c, c["gc"].astype(np.float64), c["gv"].astype(np.float64), 1, debug=True)
    assert np.abs(M1 - d["M"]).max() < 2e-6 * np.abs(d["M"]).max()
    assert np.abs(h1 - d["h"]).max() < 2e-5 * max(np.abs(d["h"]).max(), 1.0)
    assert (np.abs(M1 - M0).max(axis=(1, 2)) > 1e-3).all()
    bt.clear_body_inertia()
    assert bt.mass_matrix().tobytes() == M0.tobytes() and bt.launch_count() == L0 + 2


def test_host_device_and_pybind_sources_agree(capi, monkeypatch):
    import torch
    from raisimlib_b200 import _rsb_py
    n = 200
    rows = None
    out = {}
    for mode in ("host", "device", "raw"):
        c = _make(capi, monkeypatch, "quadruped", n, "ground", seed=53, oracles=False)
        rows = _distinct_rows(c["t"], n, 11)
        if mode == "host":
            c["bt"].set_body_inertia(rows[50:], env_begin=50); c["bt"].set_body_inertia(rows[:50])
        elif mode == "device":
            c["bt"].set_body_inertia_from(torch.from_numpy(rows).cuda())
        else:
            tr = torch.from_numpy(rows).cuda()
            assert capi.lib().rsb_batch_set_body_inertia(c["bt"].h, C.c_void_p(tr.data_ptr()), 0, n, capi.DEVICE) == 0
        for k in range(3):
            c["bt"].integrate(SUB)
        out[mode] = _outputs(c["bt"])
    _same(out["host"], out["device"], "device source: ")
    _same(out["host"], out["raw"], "ctypes device source: ")
    c = _make(capi, monkeypatch, "quadruped", n, "ground", seed=53, oracles=False)
    with pytest.raises(ValueError):
        c["bt"].set_body_inertia_from(torch.from_numpy(rows).double().cuda())
    with pytest.raises(ValueError):
        c["bt"].set_body_inertia_from(torch.from_numpy(rows[:, :, :9].copy()).cuda())
    with pytest.raises(ValueError):
        c["bt"].set_body_inertia_from(torch.from_numpy(rows).cuda().transpose(0, 1))
    with pytest.raises(ValueError):
        c["bt"].set_body_inertia_from(torch.from_numpy(rows))
    # the pybind module against the ctypes binding: same state through DLPack, same rows from the device
    monkeypatch.delenv("RSB_FORCE_WPC", raising=False); monkeypatch.setenv("RSB_FORCE_GENERIC", "0")
    path = os.path.join(RSC, "anymal_c_like.urdf")
    pb = _rsb_py.Batch(_rsb_py.Model(path), n, 0)
    bt = capi.Batch(capi.Model(path), n)
    gc = np.tile(ANYMAL_GC0.astype(np.float32), (n, 1)); gc[:, 2] = 0.54
    gc[:, 7:] += np.random.default_rng(9).uniform(-0.1, 0.1, (n, 12)).astype(np.float32)
    pb.set_ground(0.0); bt.set_ground(0.0)
    torch.from_dlpack(pb.gc()).copy_(torch.from_numpy(gc).cuda())
    bt.set_state(gc, np.zeros((n, 18), np.float32))
    tr = torch.from_numpy(rows).cuda()
    torch.cuda.synchronize()
    pb.set_body_inertia(tr.data_ptr(), 0, n); bt.set_body_inertia(rows)
    pb.integrate(SUB); bt.integrate(SUB); pb.sync()
    assert torch.from_dlpack(pb.gc()).cpu().numpy().tobytes() == bt.get_state()[0].tobytes()


def test_refusals_change_nothing(capi, monkeypatch):
    import torch
    n = 200
    L = capi.lib()
    runs = {}
    for mode in ("clean", "refused", "first_refused", "never"):
        c = _make(capi, monkeypatch, "quadruped", n, "hm", seed=57, oracles=False)
        bt = c["bt"]
        rows = _distinct_rows(c["t"], n, 13)
        if mode == "clean":
            bt.set_body_inertia(rows)
        if mode in ("refused", "first_refused"):
            if mode == "refused":
                bt.set_body_inertia(rows)
            bad = []
            for k, v in (("nan", np.nan), ("inf", np.inf)):
                r = rows.copy(); r[37, 2, 5] = v; bad.append((k, r))
            r = rows.copy(); r[120, 4, 0] = -0.5; bad.append(("negative mass", r))
            r = rows.copy(); r[7, 1, 4:] = [0.01, 0.05, 0.0, 0.01, 0.0, 0.01]; bad.append(("not PSD", r))
            r = rows.copy(); r[199, 12, 4:] = [-0.01, 0.0, 0.0, 0.02, 0.0, 0.02]; bad.append(("negative diagonal", r))
            for what, r in bad:
                for where in (capi.HOST, capi.DEVICE):
                    src = torch.from_numpy(r).cuda() if where == capi.DEVICE else r
                    ptr = C.c_void_p(src.data_ptr()) if where == capi.DEVICE else r.ctypes.data_as(C.c_void_p)
                    assert L.rsb_batch_set_body_inertia(bt.h, ptr, 0, n, where) == -1, what
                    assert b"no row changed" in L.rsb_last_error(), what
            ok = rows.ctypes.data_as(C.c_void_p)
            for begin, count, where in ((n - 1, 2, capi.HOST), (-1, 1, capi.HOST), (0, -1, capi.HOST), (0, n, 7)):
                assert L.rsb_batch_set_body_inertia(bt.h, ok, begin, count, where) == -1
        runs[mode] = []
        for k in range(3):
            bt.integrate(SUB)
            runs[mode].append(_outputs(bt))
            runs[mode][-1]["M"] = bt.mass_matrix()
    for k in range(3):
        _same(runs["clean"][k], runs["refused"][k], f"after refusals, step {k}: ")
        _same(runs["never"][k], runs["first_refused"][k], f"refused first call, step {k}: ")


def test_gym_resets_keep_the_rows(capi, monkeypatch):
    """the gym task's steps and resets leave the rows in place: after them M is that of the rows, not the model's"""
    n = 256
    g = _make(capi, monkeypatch, "quadruped", n, "ground", seed=59, oracles=False)
    rows = _distinct_rows(g["t"], n, 17)
    g["bt"].set_body_inertia(rows)
    gc_init = ANYMAL_GC0.copy(); gc_init[2] = 0.54
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
    M = g["bt"].mass_matrix()
    same, model = (_make(capi, monkeypatch, "quadruped", n, "ground", seed=59, oracles=False)["bt"] for _ in range(2))
    same.set_body_inertia(rows)
    for b in (same, model):
        b.set_state(gc, gv)
    assert M.tobytes() == same.mass_matrix().tobytes()
    assert (np.abs(M - model.mass_matrix()).max(axis=(1, 2)) > 1e-3).all()


def test_a_batch_on_another_device(capi, monkeypatch):
    """a batch on cuda:1 set while cuda:0 is current behaves as with its own device current"""
    import torch
    if torch.cuda.device_count() < 2:
        pytest.skip("needs two GPUs")
    monkeypatch.delenv("RSB_FORCE_WPC", raising=False); monkeypatch.setenv("RSB_FORCE_GENERIC", "0")
    path = os.path.join(RSC, "anymal_c_like.urdf")
    t = load_tables(path)
    n = 128
    rows = _distinct_rows(t, n, 19)
    gc = np.tile(ANYMAL_GC0.astype(np.float32), (n, 1)); gc[:, 2] = 0.54
    out = []
    for current in (0, 1):
        bt = capi.Batch(capi.Model(path), n, device=1)
        bt.set_ground(0.0); bt.set_state(gc, np.zeros((n, 18), np.float32))
        torch.cuda.set_device(current)
        bt.set_body_inertia(rows[:64])
        torch.cuda.set_device(current)
        bt.set_body_inertia_from(torch.from_numpy(rows[64:]).to("cuda:1"), env_begin=64)
        torch.cuda.set_device(current)
        M = bt.mass_matrix()
        bt.integrate(SUB)
        out.append((M.tobytes(), bt.get_state()[0].tobytes()))
    torch.cuda.set_device(0)
    assert out[0] == out[1]


def test_cpp_mass_randomization_example():
    """the raisim:: facade: getMass() / getBodyCOM_B() / getInertia() + updateMassInfo() in an upstream-shaped environment, one launch
    per control step, environment k equal to a stand-alone World with the same payload (examples/mass_randomization.cpp)"""
    exe = os.path.join(ROOT, "examples", "mass_randomization")
    if not os.path.exists(exe):
        subprocess.check_call(["make", "-C", os.path.join(ROOT, "examples")])
    out = subprocess.run([exe, os.path.join(RSC, "anymal_c_like.urdf")], capture_output=True, text=True, timeout=300)
    print(out.stdout)
    assert out.returncode == 0, out.stdout + out.stderr
