"""Per-body contact forces over a whole launch (rsb_batch_set_contact_bodies / rsb_batch_get_body_contact_forces), through the C-ABI
on an H100 (pytest -m gpu): the step kernel's accumulation over the sub-steps against tests/contact_force_ref.py on the float32 and
float64 oracles, against the contact records the kernel already writes, and the rules of the contract (launch shapes, side effects,
which launches write, slices, refusals)."""
import os
import subprocess

import numpy as np
import pytest

from conftest import ROOT, RSC
from contact_force_ref import step_with_forces
from helpers import ANYMAL_GC0, MARGIN, THRESH, launch_config
from oracle.oracle import Oracle
from oracle.self_oracle import SelfOracle
from oracle.urdf_tables import load_tables
from test_self_collision_oracle import anymal_leg_pairs, crossed_anymal

pytestmark = pytest.mark.gpu

SUB, DT = 4, 0.0025
FEET = ("LF_FOOT", "RF_FOOT", "LH_FOOT", "RH_FOOT")      # fixed to the shanks: bodies 3, 6, 9, 12 of the ANYmal-like model
# name -> robot description, RSB_FORCE_GENERIC, compiled instance (spec), base height
CASES = {"quadruped": ("anymal_c_like.urdf", False, 1, 0.56), "humanoid": ("atlas_like.urdf", False, 2, 0.95),
         "generic": ("anymal_c_like.urdf", True, 0, 0.56)}


@pytest.fixture(scope="module")
def capi():
    import torch
    assert torch.cuda.is_available(), "GPU tests need a CUDA device"
    from raisimlib_b200 import capi as c
    return c


def _make(capi, monkeypatch, name, n, terrain, seed, wpc=None, oracles=True):
    """upright robots with a small tilt and jittered joints just above the terrain, stiff PD towards targets near the nominal pose"""
    urdf, generic, spec, base_z = CASES[name]
    monkeypatch.setenv("RSB_FORCE_GENERIC", "1" if generic else "0")
    if wpc is None:
        monkeypatch.delenv("RSB_FORCE_WPC", raising=False)
    else:
        monkeypatch.setenv("RSB_FORCE_WPC", str(wpc))
    path = os.path.join(RSC, urdf)
    t = load_tables(path)
    bt = capi.Batch(capi.Model(path), n)
    cfg = launch_config(capi, bt)
    assert cfg["spec"] == spec, f"{name}: runs instance {cfg}"
    prm = dict(threshold=THRESH)
    bt.set_params(**prm)
    os_ = [Oracle(t, params=prm), Oracle(t, precision="f32", params=prm)] if oracles else []
    rng = np.random.default_rng(seed)
    if terrain == "ground":
        bt.set_ground(0.0)
        for o in os_:
            o.set_ground(0.0)
    else:
        H = (0.1 * rng.uniform(-1, 1, (49, 65))).astype(np.float32)
        bt.set_heightmap(65, 49, 12.8, 9.6, 0.1, -0.2, H)
        for o in os_:
            o.set_heightmap(65, 49, 12.8, 9.6, 0.1, -0.2, H.astype(np.float64))
    gc0 = np.zeros(t["nq"]); gc0[2] = base_z; gc0[3] = 1.0
    if t["nq"] == 19:
        gc0[7:] = ANYMAL_GC0[7:]
    gc = np.tile(gc0, (n, 1)); gc[:, :2] = rng.uniform(-2, 2, (n, 2))
    q = np.c_[np.ones(n), 0.08 * rng.standard_normal((n, 3))]
    gc[:, 3:7] = q / np.linalg.norm(q, axis=1, keepdims=True)
    gc[:, 7:] += rng.uniform(-0.15, 0.15, (n, t["nq"] - 7))
    gv = 0.3 * rng.standard_normal((n, t["nv"]))
    gc, gv = gc.astype(np.float32), gv.astype(np.float32)
    kp = np.r_[np.zeros(6), 300.0 * np.ones(t["nv"] - 6)]; kd = np.r_[np.zeros(6), 4.0 * np.ones(t["nv"] - 6)]
    pt = np.tile(gc0, (n, 1)); pt[:, 7:] += rng.uniform(-0.3, 0.3, (n, t["nq"] - 7))
    pt = pt.astype(np.float32)
    bt.set_control_mode(capi.PD_PLUS_FEEDFORWARD_TORQUE)
    bt.set_pd_gains(kp, kd)
    bt.set_pd_target(pt, np.zeros((n, t["nv"]), np.float32))
    bt.set_state(gc, gv)
    return dict(t=t, bt=bt, o=os_, gc=gc, gv=gv, kp=kp, kd=kd, pt=pt, cfg=cfg, n=n)


def _outputs(bt):
    """everything a step leaves behind besides the contact forces, for bit-identity checks"""
    gc, gv = bt.get_state()
    ct, cnt = bt.contacts()
    return dict(gc=gc, gv=gv, ct=ct.view(np.uint8), cnt=cnt, pts=bt.contact_points(), it=bt.solver_iterations(), st=bt.solver_status(),
                res=bt.solver_residual(), dv=bt.diverged(), tau=bt.generalized_force(), obs=bt.observe())


def _same(a, b, what=""):
    for k in a:
        assert np.asarray(a[k]).tobytes() == np.asarray(b[k]).tobytes(), f"{what}{k} differs"


def _scatter_records(ct, cnt, bodies, dt, substeps=1):
    """what the kernel must have stored for one sub-step, from its own contact records: float32 sums in list order, then the
    float32 reciprocal of substeps * dt"""
    n = len(cnt)
    f, s = np.zeros((n, len(bodies), 3), np.float32), np.zeros((n, len(bodies)), np.int32)
    for k in range(ct.shape[1]):
        live = k < cnt
        for j, body in enumerate(bodies):
            first = live & (ct["local_body"][:, k] == body)
            second = live & (ct["pair_index"][:, k] < 0) & (-1 - ct["pair_index"][:, k] == body)
            f[:, j] = np.where(first[:, None], f[:, j] + ct["impulse"][:, k], np.where(second[:, None], f[:, j] - ct["impulse"][:, k], f[:, j]))
            s[:, j] |= (first | second)
    scale = np.float32(1.0) / (np.float32(substeps) * np.float32(dt))
    return f * scale, s


# ---- 1: against the oracle ---------------------------------------------------------------------------------------------------------

@pytest.mark.parametrize("terrain", ["ground", "hm"])
@pytest.mark.parametrize("name", list(CASES))
def test_forces_and_steps_match_the_oracle(capi, monkeypatch, name, terrain):
    """512 environments, 4 sub-steps, every body listed.  A second batch runs the same sub-steps as four launches and shows the
    kernel's contact list of each; where those equal the float32 oracle's in every sub-step (no candidate within MARGIN of the
    surface) and every solve converged on both sides, steps_in_contact is exact, and the forces stay within the normal-impulse bound of tests/test_gpu_instances.py over dt,
    or the float32 oracle's own distance from the float64 one"""
    n = 512
    c = _make(capi, monkeypatch, name, n, terrain, seed=300 + len(name) + (terrain == "hm"))
    t, bt = c["t"], c["bt"]
    bodies = list(range(t["nb"]))
    assert len(bodies) <= 32
    bt.set_contact_bodies(bodies)
    bt.integrate(SUB)
    f, s = bt.body_contact_forces()
    kw = dict(ptarget=c["pt"].astype(np.float64), vtarget=np.zeros((n, t["nv"])), kp=c["kp"], kd=c["kd"])
    f64, s64, d64 = step_with_forces(c["o"][0], c["gc"].astype(np.float64), c["gv"].astype(np.float64), SUB, bodies, **kw)
    f32, s32, d32 = step_with_forces(c["o"][1], c["gc"].astype(np.float64), c["gv"].astype(np.float64), SUB, bodies, **kw)
    # the kernel's own list of every sub-step
    c2 = _make(capi, monkeypatch, name, n, terrain, seed=300 + len(name) + (terrain == "hm"), oracles=False)
    ok = np.ones(n, bool)
    for k in range(SUB):
        c2["bt"].integrate(1)
        pts, (_, cnt) = c2["bt"].contact_points(), c2["bt"].contacts()
        shallow = ((np.abs(d32[k]["c_depth"]) < MARGIN) & (d32[k]["c_pt"] >= 0)).any(1)
        ok &= ~shallow & (pts == d32[k]["c_pt"]).all(1) & (cnt == d32[k]["ncontacts"]) & (d32[k]["c_pt"] == d64[k]["c_pt"]).all(1)
        ok &= (d64[k]["status"] == 0) & (d32[k]["status"] == 0) & (c2["bt"].solver_status() == 0)
    assert c2["bt"].get_state()[0].tobytes() == bt.get_state()[0].tobytes()
    assert ok.mean() > 0.7, f"only {ok.sum()} of {n} environments have the oracle's contact lists in every sub-step"
    assert (s[ok] == s32[ok]).all()
    assert s.max() == SUB and (s > 0).any(0).sum() >= 2 and ((s > 0) & (s < SUB)).any()
    scale = max(1.0, max(np.abs(d["c_lambda"][:, :, 2]).max() for d in d64)) / DT
    e, e32 = np.abs(f - f64)[ok].max((1, 2)), np.abs(f32 - f64)[ok].max((1, 2))
    print(f"{name} {terrain}: envs compared {ok.sum()}, bodies touched {int((s > 0).any(0).sum())}, force scale {scale:.0f} N, |f - f64| median "
          f"{np.median(e):.2e} p99 {np.quantile(e, .99):.2e} max {e.max():.2e}; f32 oracle median {np.median(e32):.2e} p99 {np.quantile(e32, .99):.2e} max {e32.max():.2e}")
    assert np.isfinite(f).all()
    assert np.median(e) < max(1e-4 * scale, 3 * np.median(e32))
    assert np.quantile(e, 0.99) < max(1e-4 * scale, 5 * np.quantile(e32, 0.99))
    assert e.max() < max(0.1 * scale, 5 * e32.max())       # the tail: one environment in 512 whose slip direction differs in a sub-step


# ---- 2, 3: against what the kernel already reports ------------------------------------------------------------------------------------

@pytest.mark.parametrize("name", list(CASES))
def test_one_sub_step_equals_the_scatter_of_the_contact_records(capi, monkeypatch, name):
    c = _make(capi, monkeypatch, name, 512, "hm", seed=41, oracles=False)
    bt, bodies = c["bt"], list(range(c["t"]["nb"]))
    bt.set_contact_bodies(bodies)
    for k in range(3):
        bt.integrate(1)
        f, s = bt.body_contact_forces()
        ct, cnt = bt.contacts()
        fr, sr = _scatter_records(ct, cnt, bodies, DT)
        assert cnt.sum() > 100
        assert (s == sr).all()
        assert f.tobytes() == fr.tobytes(), f"sub-step {k}: largest difference {np.abs(f - fr).max():.3e}"


def test_four_launches_of_one_sub_step_add_up_to_one_launch_of_four(capi, monkeypatch):
    a = _make(capi, monkeypatch, "quadruped", 512, "hm", seed=43, oracles=False)
    b = _make(capi, monkeypatch, "quadruped", 512, "hm", seed=43, oracles=False)
    feet = [a["bt"].model.body_index(x) for x in FEET]
    bodies = list(range(13))
    a["bt"].set_contact_bodies(bodies); b["bt"].set_contact_bodies(bodies)
    a["bt"].integrate(SUB)
    fa, sa = a["bt"].body_contact_forces()
    fs, ss = np.zeros_like(fa, dtype=np.float64), np.zeros_like(sa)
    for k in range(SUB):
        b["bt"].integrate(1)
        f, s = b["bt"].body_contact_forces()
        fs += f; ss += s
    _same(_outputs(a["bt"]), _outputs(b["bt"]))
    assert (ss == sa).all() and sa[:, feet].max() == SUB
    assert np.abs(fs / SUB - fa).max() < 4e-6 * max(1.0, np.abs(fa).max())


# ---- 4: self contacts -------------------------------------------------------------------------------------------------------------------

def test_self_contacts_act_on_both_bodies_with_opposite_forces(capi, monkeypatch):
    monkeypatch.delenv("RSB_FORCE_WPC", raising=False); monkeypatch.setenv("RSB_FORCE_GENERIC", "0")
    path = os.path.join(RSC, "anymal_c_like.urdf")
    t = load_tables(path)
    n, pairs, bodies = 256, anymal_leg_pairs(), list(range(13))
    rng = np.random.default_rng(77)
    kp = np.r_[np.zeros(6), 100.0 * np.ones(12)]; kd = np.r_[np.zeros(6), 2.0 * np.ones(12)]
    for terrain in (False, True):
        prm = dict(threshold=THRESH) if terrain else dict(threshold=THRESH, gz=0.0)
        bt = capi.Batch(capi.Model(path), n)
        bt.set_params(threshold=THRESH)
        if not terrain:
            bt.set_params(gravity=(0.0, 0.0, 0.0))
        o = SelfOracle(t, params=prm)
        bt.set_self_collision(pairs); o.set_self_collision(pairs)
        assert launch_config(capi, bt)["spec"] == 0
        if terrain:
            bt.set_ground(0.0); o.set_ground(0.0)
        gc = crossed_anymal(n, rng, z=0.45 if terrain else 1.0).astype(np.float32)
        gv = (0.3 * rng.standard_normal((n, 18))).astype(np.float32)
        pt = gc.copy(); pt[:, [7, 13]] -= 0.5; pt[:, [10, 16]] += 0.5
        bt.set_control_mode(capi.PD_PLUS_FEEDFORWARD_TORQUE); bt.set_pd_gains(kp, kd)
        bt.set_pd_target(pt, np.zeros((n, 18), np.float32)); bt.set_state(gc, gv)
        bt.set_contact_bodies(bodies)
        bt.integrate(SUB)
        f, s = bt.body_contact_forces()
        ct, cnt = bt.contacts()
        f64, s64, d64 = step_with_forces(o, gc.astype(np.float64), gv.astype(np.float64), SUB, bodies, ptarget=pt.astype(np.float64),
                                         vtarget=np.zeros((n, 18)), kp=kp, kd=kd)
        scale = max(1.0, np.abs(f64).max())
        assert (s > 0).sum() > n and np.isfinite(f).all()
        if not terrain:
            assert all((d["c_pair"][d["c_pt"] >= 0] < 0).all() for d in d64)
            assert np.abs(f.sum(1)).max() < 2e-6 * scale                     # action = reaction, to float32 rounding of the lanes' sums
            one = (s.sum(1) == 2 * SUB) & ((s > 0).sum(1) == 2)               # one pair in contact throughout: exactly opposite
            assert one.sum() > 3
            for e in np.where(one)[0]:
                i, j = np.where(s[e] > 0)[0]
                assert (f[e, i] == -f[e, j]).all()
        same = np.all([(d["status"] == 0) for d in d64], 0) & (s == s64).all(1)
        e = np.abs(f - f64)[same].max((1, 2))
        print(f"self contacts, terrain {terrain}: envs compared {same.sum()} of {n}, |f - f64| median {np.median(e):.2e} p99 {np.quantile(e, .99):.2e} of {scale:.0f} N")
        assert same.mean() > 0.7 and np.median(e) < 1e-4 * scale and np.quantile(e, 0.99) < 2e-2 * scale
        del bt


# ---- 5: no side effects; who writes ---------------------------------------------------------------------------------------------------

def test_listing_bodies_changes_nothing_else_and_only_stepping_launches_write(capi, monkeypatch):
    runs = {}
    for mode in ("never", "listed", "cleared"):
        c = _make(capi, monkeypatch, "quadruped", 300, "hm", seed=51, oracles=False)
        bt = c["bt"]
        if mode != "never":
            bt.set_contact_bodies(list(range(13)))
            f0, s0 = bt.body_contact_forces()
            assert not f0.any() and not s0.any()                              # zero until the first stepping launch
        if mode == "cleared":
            bt.integrate(SUB); bt.set_state(c["gc"], c["gv"]); bt.set_contact_bodies([])
        out = []
        for k in range(10):
            bt.integrate(SUB)
            out.append(_outputs(bt))
            if mode == "listed":
                f, s = bt.body_contact_forces()
                bt.body_poses(); bt.integrate1(); bt.update_kinematics()
                bt.set_frames([0, 3], np.zeros((2, 3))); bt.frame_states()
                f2, s2 = bt.body_contact_forces()
                assert f.tobytes() == f2.tobytes() and s.tobytes() == s2.tobytes() and s.any()
        runs[mode] = out
    for mode in ("listed", "cleared"):
        for k in range(10):
            _same(runs["never"][k], runs[mode][k], f"{mode}, control step {k}: ")


# ---- 6: launch shapes -----------------------------------------------------------------------------------------------------------------

@pytest.mark.parametrize("name", ["quadruped", "humanoid"])
def test_every_launch_shape_gives_the_same_forces(capi, monkeypatch, name):
    """every CTA size that fits, the sub-step barrier and the paired stage A on and off; the batch ends on a partly filled round"""
    n = 4500 if name == "quadruped" else 2300
    ref, taken = None, []
    shapes = [(None, "1", "1")] + [(w, "1", "1") for w in (28, 16, 14, 8, 4, 1)] + [(None, "0", "1"), (None, "1", "0")]
    for wpc, barrier, pair in shapes:
        monkeypatch.setenv("RSB_SUBSTEP_BARRIER", barrier); monkeypatch.setenv("RSB_PAIR_STAGE_A", pair)
        c = _make(capi, monkeypatch, name, n, "hm", seed=61, wpc=wpc, oracles=False)
        if wpc is not None and c["cfg"]["wpc"] != wpc:
            continue                                                          # did not fit
        taken.append(c["cfg"]["wpc"])
        c["bt"].set_contact_bodies(list(range(c["t"]["nb"])))
        for k in range(2):
            c["bt"].integrate(SUB)
        f, s = c["bt"].body_contact_forces()
        if ref is None:
            ref = (f, s)
            T = c["cfg"]["wpc"] * c["cfg"]["grid"]
            assert n % T != 0 and s.any()
        assert f.tobytes() == ref[0].tobytes() and s.tobytes() == ref[1].tobytes(), f"{name}: differs at wpc {wpc} barrier {barrier} pairing {pair}"
        del c
    assert len(set(taken)) >= 5


# ---- 7: control_step and gym_step ---------------------------------------------------------------------------------------------------

def test_control_step_and_gym_step_fill_the_outputs(capi, monkeypatch):
    import torch
    a = _make(capi, monkeypatch, "quadruped", 256, "ground", seed=71, oracles=False)
    b = _make(capi, monkeypatch, "quadruped", 256, "ground", seed=71, oracles=False)
    feet = [3, 6, 9, 12]
    a["bt"].set_contact_bodies(feet); b["bt"].set_contact_bodies(feet)
    a["bt"].integrate(SUB)
    pin_t = torch.from_numpy(b["pt"]).pin_memory(); pin_o = torch.empty((256, b["bt"].ob_dim()), dtype=torch.float32).pin_memory()
    b["bt"].control_step(pin_t, SUB, pin_o)
    fa, sa = a["bt"].body_contact_forces(); fb, sb = b["bt"].body_contact_forces()
    assert fa.tobytes() == fb.tobytes() and sa.tobytes() == sb.tobytes() and sa.any()
    # gym task: large actions fold robots up, they terminate and are reset; their forces are those of the step that ended them
    n = 256
    g = _make(capi, monkeypatch, "quadruped", n, "ground", seed=72, oracles=False)
    gc_init = ANYMAL_GC0.copy(); gc_init[2] = 0.54
    bodies, nonfoot = list(range(13)), np.setdiff1d(np.arange(13), feet)
    g["bt"].set_contact_bodies(bodies)
    g["bt"].gym_configure(gc_init, np.zeros(18), gc_init[7:], 0.6 * np.ones(12), feet)
    g["bt"].gym_reset()
    rng = np.random.default_rng(5)
    obs = np.empty((n, 34), np.float32); rew = np.empty(n, np.float32); done = np.empty(n, np.uint8)
    terminated = 0
    base = rng.normal(0, 1.5, (n, 12))                            # persistent offsets: many robots fold up and terminate
    for k in range(60):
        sub = 1 if k % 2 else SUB
        g["bt"].gym_step((base + rng.normal(0, 0.3, (n, 12))).astype(np.float32), sub, obs, rew, done)
        f, s = g["bt"].body_contact_forces()
        ct, cnt = g["bt"].contacts()
        if sub == 1:        # one sub-step: the contact records of the launch tell the whole story, reset environments included
            fr, sr = _scatter_records(ct, cnt, bodies, DT)
            assert f.tobytes() == fr.tobytes() and s.tobytes() == sr.tobytes()
        d = done == 1
        terminated += int(d.sum())
        assert (s[d][:, nonfoot] > 0).any(1).all() and (s <= sub).all()       # a terminated environment shows what ended it
        assert (g["bt"].get_state()[0][d] == gc_init.astype(np.float32)).all()                 # ... although its state is the reset one
    assert terminated > 10


# ---- 8: slices, destinations, refusals ------------------------------------------------------------------------------------------------

def test_slices_destinations_and_refusals(capi, monkeypatch):
    import ctypes as C
    import torch
    c = _make(capi, monkeypatch, "quadruped", 200, "hm", seed=81, oracles=False)
    bt, L = c["bt"], capi.lib()
    with pytest.raises(capi.RsbError, match="no contact bodies"):
        bt.ncontact_bodies = 4; bt.body_contact_forces()
    feet = [3, 6, 9, 12]
    bt.set_contact_bodies(feet)
    bt.integrate(SUB)
    f, s = bt.body_contact_forces()
    assert f.shape == (200, 4, 3) and s.shape == (200, 4) and s.any()
    f1, s1 = bt.body_contact_forces(37, 100)
    assert f1.tobytes() == f[37:137].tobytes() and s1.tobytes() == s[37:137].tobytes()
    tf, ts = torch.zeros((100, 4, 3), device="cuda"), torch.zeros((100, 4), dtype=torch.int32, device="cuda")
    launches = bt.launch_count()
    bt.body_contact_forces_into(tf, ts, 37, 100); bt.sync()
    assert bt.launch_count() == launches                                      # a copy, no kernel
    assert tf.cpu().numpy().tobytes() == f1.tobytes() and ts.cpu().numpy().tobytes() == s1.tobytes()
    tf.zero_(); ts.fill_(-1)
    bt.body_contact_forces_into(force=tf, env_begin=37, env_count=100); bt.sync()
    assert tf.cpu().numpy().tobytes() == f1.tobytes() and (ts.cpu().numpy() == -1).all()           # a NULL output is skipped
    bt.body_contact_forces_into(steps=ts, env_begin=37, env_count=100); bt.sync()
    assert ts.cpu().numpy().tobytes() == s1.tobytes()
    with pytest.raises(ValueError):
        bt.body_contact_forces_into(steps=torch.zeros((100, 4), device="cuda"), env_begin=37, env_count=100)     # float32 steps
    # refusals change nothing
    arr = lambda v: np.asarray(v, np.int32).ctypes.data_as(C.c_void_p)
    for body, cnt in ((arr([0] * 33), 33), (arr([0]), -1), (None, 2), (arr([0, 13]), 2), (arr([-1]), 1)):
        assert L.rsb_batch_set_contact_bodies(bt.h, body, cnt) == -1 and L.rsb_last_error()
    assert L.rsb_batch_get_body_contact_forces(bt.h, 150, 100, None, None, 0) == -1
    f2, s2 = bt.body_contact_forces()
    assert f2.tobytes() == f.tobytes() and s2.tobytes() == s.tobytes()
    d = _make(capi, monkeypatch, "quadruped", 200, "hm", seed=81, oracles=False)
    d["bt"].set_contact_bodies(feet)
    for x in (bt, d["bt"]):
        x.set_state(c["gc"], c["gv"]); x.integrate(SUB)
    fa, sa = bt.body_contact_forces(); fb, sb = d["bt"].body_contact_forces()
    assert fa.tobytes() == fb.tobytes() and sa.tobytes() == sb.tobytes()
    # a new list reads zero until the next step, then holds the new bodies in its own tight layout
    bt.set_contact_bodies_by_name(["base", "LF_FOOT"])
    f3, s3 = bt.body_contact_forces()
    assert f3.shape == (200, 2, 3) and not f3.any() and not s3.any()
    bt.set_state(c["gc"], c["gv"]); bt.integrate(SUB)
    f4, s4 = bt.body_contact_forces()
    assert f4[:, 1].tobytes() == np.ascontiguousarray(fa[:, 0]).tobytes() and (s4[:, 1] == sa[:, 0]).all()


# ---- 9: the pybind module and the C++ facade ------------------------------------------------------------------------------------------

def test_pybind_module_fills_torch_tensors(capi, monkeypatch):
    import torch
    from raisimlib_b200 import _rsb_py
    monkeypatch.delenv("RSB_FORCE_WPC", raising=False); monkeypatch.setenv("RSB_FORCE_GENERIC", "0")
    path = os.path.join(RSC, "anymal_c_like.urdf")
    n, feet = 128, [3, 6, 9, 12]
    pb = _rsb_py.Batch(_rsb_py.Model(path), n, 0)
    bt = capi.Batch(capi.Model(path), n)
    gc = np.tile(ANYMAL_GC0.astype(np.float32), (n, 1)); gc[:, 2] = 0.54
    gc[:, 7:] += np.random.default_rng(9).uniform(-0.1, 0.1, (n, 12)).astype(np.float32)
    pb.set_ground(0.0); bt.set_ground(0.0)
    torch.from_dlpack(pb.gc()).copy_(torch.from_numpy(gc).cuda())
    bt.set_state(gc, np.zeros((n, 18), np.float32))
    pb.set_contact_bodies(feet); bt.set_contact_bodies(feet)
    torch.cuda.synchronize()
    pb.integrate(SUB); bt.integrate(SUB)
    tf, ts = torch.zeros((n, 4, 3), device="cuda"), torch.zeros((n, 4), dtype=torch.int32, device="cuda")
    pb.body_contact_forces(tf.data_ptr(), ts.data_ptr()); pb.sync()
    f, s = bt.body_contact_forces()
    assert s.any() and tf.cpu().numpy().tobytes() == f.tobytes() and ts.cpu().numpy().tobytes() == s.tobytes()


def test_cpp_contact_forces_example():
    """the raisim:: facade: setContactBodies / getBodyContactForce / getBodyContactSteps stand-alone and inside
    VectorizedEnvironment, one launch per control step (examples/contact_forces.cpp)"""
    exe = os.path.join(ROOT, "examples", "contact_forces")
    if not os.path.exists(exe):
        subprocess.check_call(["make", "-C", os.path.join(ROOT, "examples")])
    out = subprocess.run([exe, os.path.join(RSC, "anymal_c_like.urdf")], capture_output=True, text=True, timeout=300)
    print(out.stdout)
    assert out.returncode == 0, out.stdout + out.stderr


# ---- 10: a known answer ---------------------------------------------------------------------------------------------------------------

def test_standing_robots_feet_carry_the_weight(capi, monkeypatch):
    monkeypatch.delenv("RSB_FORCE_WPC", raising=False); monkeypatch.setenv("RSB_FORCE_GENERIC", "0")
    path = os.path.join(RSC, "anymal_c_like.urdf")
    t = load_tables(path)
    n = 64
    bt = capi.Batch(capi.Model(path), n)
    bt.set_ground(0.0)
    gc = np.tile(ANYMAL_GC0.astype(np.float32), (n, 1)); gc[:, 2] = 0.54
    gc[:, 7:] += np.random.default_rng(4).uniform(-0.05, 0.05, (n, 12)).astype(np.float32)
    kp = np.r_[np.zeros(6), 300.0 * np.ones(12)]; kd = np.r_[np.zeros(6), 8.0 * np.ones(12)]
    bt.set_control_mode(capi.PD_PLUS_FEEDFORWARD_TORQUE); bt.set_pd_gains(kp, kd)
    bt.set_pd_target(gc, np.zeros((n, 18), np.float32)); bt.set_state(gc, np.zeros((n, 18), np.float32))
    bt.set_contact_bodies_by_name(FEET)
    for k in range(200):                                                      # 2 s: settled
        bt.integrate(SUB)
    f, s = bt.body_contact_forces()
    weight = t["mass"].sum() * 9.81
    assert (s == SUB).all()
    assert np.abs(f[:, :, 2].sum(1) - weight).max() < 0.02 * weight
    assert np.abs(f[:, :, :2].sum(1)).max() < 0.02 * weight
