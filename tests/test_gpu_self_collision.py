"""Self-collision on the GPU (run on an H100: pytest -m gpu): the generic instance of the step kernel with pairs enabled against the
float32 / float64 oracle, bit-identity where nothing may change, the refusals of rsb_batch_set_self_collision, and the facade.  Every
test reads back through rsb_internal_launch_instance which instance ran (tests/helpers.py launch_config)."""
import ctypes
import os
import subprocess

import numpy as np
import pytest

from helpers import ANYMAL_GC0, MAX32, THRESH, ROW_BIAS, setup_batch, index_parity, launch_config, check_restitution_split
from test_self_collision_oracle import anymal_leg_pairs, crossed_anymal
from oracle.self_oracle import SelfOracle, self_pair_tables
from oracle.urdf_tables import load_tables

pytestmark = pytest.mark.gpu

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
RSC = os.path.join(ROOT, "raisimlib_b200", "rsc")
# Atlas-like: thighs, knee spheres against each other, against the other thigh and the other foot; hands against the torso, the pelvis
# and each other (collision bodies: 0 pelvis box, 1 utorso box, 2 head, 4 / 6 hand spheres, 7 / 10 thigh capsules, 8 / 11 knee
# spheres, 9 / 12 foot boxes)
ATLAS_PAIRS = [(7, 10), (8, 11), (8, 10), (11, 7), (8, 12), (11, 9), (4, 1), (6, 1), (4, 0), (6, 0), (4, 6), (2, 4), (2, 6)]
SPEC_GENERIC = 0


@pytest.fixture(scope="module")
def capi():
    import torch
    assert torch.cuda.is_available(), "GPU tests need a CUDA device"
    from raisimlib_b200 import capi as c
    return c


def _env(monkeypatch, generic=False, wpc=None):
    monkeypatch.setenv("RSB_FORCE_GENERIC", "1" if generic else "0")
    if wpc is None:
        monkeypatch.delenv("RSB_FORCE_WPC", raising=False)
    else:
        monkeypatch.setenv("RSB_FORCE_WPC", str(wpc))


def _outputs(bt):
    """everything a step leaves behind, for bit-identity checks"""
    gc, gv = bt.get_state()
    ct, cnt = bt.contacts()
    return dict(gc=gc, gv=gv, ct=ct.view(np.uint8), cnt=cnt, pts=bt.contact_points(), it=bt.solver_iterations(), st=bt.solver_status(),
                res=bt.solver_residual(), tau=bt.generalized_force())


def _same(a, b):
    for k in a:
        assert np.array_equal(np.asarray(a[k]).view(np.uint8), np.asarray(b[k]).view(np.uint8)), f"{k} differs"


def _crossed(name, t, n, rng, z):
    """ANYmal-like with its legs crossed at the hips; Atlas-like with every joint up to 1.3 rad off zero (legs crossed, hands on the
    torso in many environments); both low enough to lie on the terrain as well"""
    if name == "anymal":
        gc = crossed_anymal(n, rng, z=z)
        q = np.c_[np.ones(n), 0.3 * rng.standard_normal((n, 3))]
    else:
        gc = np.zeros((n, t["nq"])); gc[:, 2] = z
        gc[:, 7:] = rng.uniform(-1.3, 1.3, (n, t["nq"] - 7))
        q = np.c_[np.ones(n), 0.3 * rng.standard_normal((n, 3))]
    gc[:, :2] = rng.uniform(-2, 2, (n, 2))
    gc[:, 3:7] = q / np.linalg.norm(q, axis=1, keepdims=True)
    gv = 0.3 * rng.standard_normal((n, t["nv"]))
    return gc.astype(np.float32).astype(np.float64), gv.astype(np.float32).astype(np.float64)


CASES = {"anymal": ("anymal_c_like.urdf", anymal_leg_pairs(), 0.45), "atlas": ("atlas_like.urdf", ATLAS_PAIRS, 0.75)}


def _setup(capi, monkeypatch, name, terrain, n, seed, params=None):
    """a batch with the case's pairs and the float64 / float32 self-collision oracles on the same terrain (a random 65 x 49 map for
    "hm"), the robots crossed (_crossed), joint torques zero"""
    urdf, pairs, z = CASES[name]
    _env(monkeypatch)
    path = os.path.join(RSC, urdf)
    t = load_tables(path)
    bt = capi.Batch(capi.Model(path), n)
    prm = dict(threshold=THRESH, **(params or {}))
    o64, o32 = SelfOracle(t, params=prm), SelfOracle(t, precision="f32", params=prm)
    bt.set_params(**prm)
    rng = np.random.default_rng(seed)
    if terrain == "ground":
        for o in (o64, o32):
            o.set_ground(0.0)
        bt.set_ground(0.0)
    else:
        xs, ys = 65, 49
        H = (0.1 * rng.uniform(-1, 1, (ys, xs))).astype(np.float32)
        for o in (o64, o32):
            o.set_heightmap(xs, ys, 12.8, 9.6, 0.1, -0.2, H.astype(np.float64))
        bt.set_heightmap(xs, ys, 12.8, 9.6, 0.1, -0.2, H)
    bt.set_control_mode(capi.FORCE_AND_TORQUE)
    bt.set_self_collision(pairs)
    for o in (o64, o32):
        o.set_self_collision(pairs)
    cfg = launch_config(capi, bt)
    assert cfg["spec"] == SPEC_GENERIC, f"pairs enabled: the generic instance must run, got {cfg}"
    gc, gv = _crossed(name, t, n, np.random.default_rng(seed + 1), z)
    bt.set_state(gc.astype(np.float32), gv.astype(np.float32))
    return t, bt, o64, o32, gc, gv, cfg


# ---- 1 / 2: nothing changes where nothing may ---------------------------------------------------------------------------------

def test_clearing_pairs_restores_default_instance(capi, monkeypatch):
    """enabling pairs and clearing them again (n = 0) gives back the default instance and bit-identical results, whatever the order in
    which the terrain friction, the pairs and the PD gains were set around them"""
    _env(monkeypatch)
    kp, kd = np.r_[np.zeros(6), 80.0 * np.ones(12)], np.r_[np.zeros(6), 2.0 * np.ones(12)]
    orders = [("friction", "gains"), ("friction", "pairs", "gains", "clear"), ("pairs", "gains", "friction", "clear")]
    runs = []
    for order in orders:
        t, bt, _, _, gc, gv, tau = setup_batch(capi, "anymal_c_like.urdf", 512, 7, terrain="hm", tau_scale=20.0)
        bt.set_control_mode(capi.PD_PLUS_FEEDFORWARD_TORQUE)
        bt.set_pd_target(np.tile(ANYMAL_GC0, (512, 1)).astype(np.float32), np.zeros((512, 18), np.float32))
        before = launch_config(capi, bt)
        for step in order:
            if step == "friction":
                bt.set_collision_friction(4, 0.5)
            elif step == "gains":
                bt.set_pd_gains(kp, kd)
            elif step == "pairs":
                bt.set_self_collision(anymal_leg_pairs())
            else:
                assert launch_config(capi, bt)["spec"] == SPEC_GENERIC
                bt.set_self_collision([])
        cfg = launch_config(capi, bt)
        assert cfg == before and cfg["spec"] == 1, order
        bt.integrate(4)
        bt.integrate(4)
        runs.append(_outputs(bt))
    for order, run in zip(orders[1:], runs[1:]):
        print("compared:", order)
        _same(runs[0], run)


def test_unreachable_pairs_bit_identical_to_generic(capi, monkeypatch):
    """pairs that cannot touch (standing quadrupeds, feet across the body, thighs side by side): bit-identical to the forced-generic
    instance without pairs"""
    far = [(4, 16), (8, 12), (4, 12), (8, 16), (2, 6), (10, 14)]
    runs = []
    for with_pairs in (False, True):
        _env(monkeypatch, generic=True)
        t, bt, _, _, _, _, _ = setup_batch(capi, "anymal_c_like.urdf", 1024, 21, terrain="hm", tau_scale=0.0)
        rng = np.random.default_rng(22)
        gc = np.tile(ANYMAL_GC0, (1024, 1)); gc[:, :2] = rng.uniform(-2, 2, (1024, 2)); gc[:, 2] = 0.56
        gc[:, 7:] += rng.uniform(-0.1, 0.1, (1024, 12))
        bt.set_state(gc.astype(np.float32), (0.2 * rng.standard_normal((1024, 18))).astype(np.float32))
        bt.set_control_mode(capi.PD_PLUS_FEEDFORWARD_TORQUE)
        bt.set_pd_gains(np.r_[np.zeros(6), 300.0 * np.ones(12)], np.r_[np.zeros(6), 8.0 * np.ones(12)])
        bt.set_pd_target(np.tile(ANYMAL_GC0, (1024, 1)).astype(np.float32), np.zeros((1024, 18), np.float32))
        if with_pairs:
            bt.set_self_collision(far)
        assert launch_config(capi, bt)["spec"] == SPEC_GENERIC
        for _ in range(5):
            bt.integrate(4)
        out = _outputs(bt)
        ct, _ = bt.contacts()
        assert (ct["pair_index"] >= -1).all()                 # no self contact was ever recorded in the last step
        runs.append(out)
    _same(runs[0], runs[1])


# ---- 3 / 4: against the oracle ---------------------------------------------------------------------------------------------------

@pytest.mark.parametrize("terrain", ["ground", "hm"])
@pytest.mark.parametrize("name", list(CASES))
def test_self_contact_lists_match_oracle(capi, monkeypatch, name, terrain):
    """contact lists (count, bodies, pair index, candidate ids) bit-exact against the float32 oracle outside the 2e-6 m margin, with
    terrain and self contacts mixed and more than 8 hits in some environments; depth, normal and position against the float64 oracle at
    the narrow-phase tolerances of DESIGN section 5"""
    n = 512
    t, bt, o64, o32, gc, gv, cfg = _setup(capi, monkeypatch, name, terrain, n, seed=300 + (terrain == "hm"))
    bt.integrate1()
    ct, cnt = bt.contacts(); pts = bt.contact_points()
    zero = np.zeros((n, t["nv"]))
    d32 = o32.step(gc.copy(), gv.copy(), tau_ff=zero, debug=True)
    d64 = o64.step(gc.copy(), gv.copy(), tau_ff=zero, debug=True)
    self_ref = (d64["c_pair"] < 0) & (d64["c_pt"] >= 0)
    terr_ref = (d64["c_pair"] >= 0) & (d64["c_pt"] >= 0)
    mixed = (self_ref.any(1) & terr_ref.any(1)).sum()
    print(f"{name} {terrain}: self contacts {int(self_ref.sum())} in {int(self_ref.any(1).sum())} envs, mixed envs {int(mixed)}, "
          f"envs at the 8-contact cap {int((d64['ncontacts'] == 8).sum())}")
    assert self_ref.sum() > n // 4 and mixed > 10
    assert (d64["ncontacts"] == 8).any() or (name, terrain) == ("anymal", "ground")     # more than 8 hits: the ranking keeps the deepest
    hard = index_parity(pts, cnt, d32, f"{name} {terrain} self")
    assert hard.sum() <= (0 if terrain == "ground" else 1)
    same = (pts == d32["c_pt"]).all(1) & (cnt == d32["ncontacts"])
    live = same[:, None] & (d64["c_pt"] >= 0) & (pts == d64["c_pt"])
    assert np.array_equal(ct["local_body"][live], d32["c_body"][live]) and np.array_equal(ct["pair_index"][live], d32["c_pair"][live])
    sl = live & (d64["c_pair"] < 0)
    ed = np.abs(ct["depth"] - d64["c_depth"])[sl]
    en = np.abs(ct["normal"] - d64["c_normal"]).max(2)[sl]
    ep = np.abs(ct["position"] - d64["c_pos"]).max(2)[sl]
    # the normal is a difference of two float32 points divided by their distance: 2e-6 + 3e-6 / distance (DESIGN section 5)
    idesc, geo = self_pair_tables(t, CASES[name][1])
    j = (d64["c_pt"] - t["npts"])[sl]
    dist = np.maximum(geo[j, 21] + geo[j, 22] - d64["c_depth"][sl], 1e-4)
    print(f"   self contacts compared {int(sl.sum())}: depth {ed.max():.1e}, normal {en.max():.1e} (x distance {(en * dist).max():.1e}), "
          f"position {ep.max():.1e}")
    assert ed.max() < 5e-6 and (en < 2e-6 + 3e-6 / dist).all() and ep.max() < 2e-5


def _complementarity(t, ct, cnt, pts, d64, Jt, v_after, conv, mu=0.8):
    """Signorini and Coulomb on every self contact of the GPU result: normal impulse >= 0, inside the friction cone, and a contact that
    pushes does not approach (J_n v+ >= 0, evaluated with the oracle's Jacobian at the start state)"""
    worst_cone, worst_sig = 0.0, 0.0
    for e in np.where(conv)[0]:                       # converged solves (not the compliant fallback)
        for k in range(cnt[e]):
            if ct["pair_index"][e, k] >= 0 or pts[e, k] != d64["c_pt"][e, k]:
                continue
            nrm = ct["normal"][e, k]; imp = ct["impulse"][e, k]
            ln = imp @ nrm; lt = np.linalg.norm(imp - ln * nrm)
            assert ln >= -1e-6
            worst_cone = max(worst_cone, lt - mu * ln)
            if ln > 1e-3 and k < d64["ncontacts"][e]:
                vn = Jt[e][:, 3 * k + 2] @ v_after[e]
                worst_sig = max(worst_sig, -vn)
    return worst_cone, worst_sig


@pytest.mark.parametrize("name,terrain,bias", [pytest.param(name, terrain, None, id=f"{name}-{terrain}") for name in CASES for terrain in ("ground", "hm")] +
                         [pytest.param("atlas", "ground", dict(ROW_BIAS, rest_threshold=0.1), id="atlas-ground-bias")])   # some self contacts beyond it
def test_self_collision_step_and_trajectory(capi, monkeypatch, name, terrain, bias):
    """one step and 10 steps against the float64 oracle within the bounds of tests/test_gpu_instances.py, Signorini and Coulomb on every
    self contact (bias: with ERP and restitution, which a self contact takes on the difference of its two halves)"""
    n = 256
    t, bt, o64, o32, gc, gv, cfg = _setup(capi, monkeypatch, name, terrain, n, seed=400 + (terrain == "hm"), params=bias)
    bt.set_control_mode(capi.FORCE_AND_TORQUE)
    bt.set_generalized_force(np.zeros((n, t["nv"]), np.float32))
    zero = np.zeros((n, t["nv"]))
    bt.integrate(1)
    g1, v1 = bt.get_state(); ct, cnt = bt.contacts(); pts = bt.contact_points(); st = bt.solver_status()
    a, b = gc.copy(), gv.copy()
    d = o64.step(a, b, tau_ff=zero, debug=True)
    c, e_ = gc.copy(), gv.copy()
    o32.step(c, e_, tau_ff=zero)
    same = (pts == d["c_pt"]).all(1)
    conv = same & (st == 0) & (d["status"] == 0)
    assert ((d["c_pair"] < 0) & (d["c_pt"] >= 0))[conv].sum() > n // 8
    ev = np.abs(v1 - b)[conv]; e32 = np.abs(e_ - b)[conv]
    scale_v = 1.0 + np.abs(b[conv])
    _, pj, Jt = o64.contact_jacobians(gc)
    assert np.array_equal(pj, d["c_pt"])
    if bias:
        vn = np.where(d["c_pt"] >= 0, np.einsum("evk,ev->ek", Jt[:, :, 2::3], gv), np.nan)       # terrain and self contacts
        check_restitution_split(vn, bias["rest_threshold"])
        assert (np.isfinite(vn) & (d["c_pair"] < 0) & (vn < -bias["rest_threshold"])).sum() >= 5
    worst_cone, worst_sig = _complementarity(t, ct, cnt, pts, d, Jt, v1.astype(np.float64), conv)
    bt.integrate(9)
    gN, _ = bt.get_state()
    o64.step(a, b, n_steps=9, tau_ff=zero)
    o32.step(c, e_, n_steps=9, tau_ff=zero)
    e = np.abs(gN - a).max(1); ef = np.abs(c - a).max(1)
    print(f"{name} {terrain}: converged {100 * conv.mean():.0f} %, 1 step gv err median {np.median(ev.max(1)):.1e} (f32 oracle "
          f"{np.median(e32.max(1)):.1e}), cone excess {worst_cone:.1e}, approach speed {worst_sig:.1e}; 10 steps gc err median {np.median(e):.1e} "
          f"p99 {np.quantile(e, .99):.1e} (f32 oracle p99 {np.quantile(ef, .99):.1e})")
    assert conv.mean() > 0.8
    assert np.median(ev.max(1)) < max(2e-5, 3 * np.median(e32.max(1)))
    assert np.max(ev / scale_v) < max(5e-3, 3 * np.max(e32 / scale_v))
    assert worst_cone < 1e-4 and worst_sig < 1e-3
    assert np.median(e) < max(2e-5, 3 * np.median(ef))
    assert np.quantile(e, 0.9) < max(1e-3, 10 * np.quantile(ef, 0.9))


# ---- 5: momentum ---------------------------------------------------------------------------------------------------------------

def test_self_contacts_conserve_momentum_gpu(capi, monkeypatch):
    """zero gravity, no terrain, legs driven into each other: the self contacts change the velocity (against the same step without
    pairs) but not M[0:6] v, linear and angular momentum; the bound is the float32 oracle's own error on the same problem, times 10"""
    n = 256
    _env(monkeypatch)
    t = load_tables(os.path.join(RSC, "anymal_c_like.urdf"))
    rng = np.random.default_rng(8)
    gc = crossed_anymal(n, rng).astype(np.float32); gv = (0.3 * rng.standard_normal((n, t["nv"]))).astype(np.float32)
    kp = np.r_[np.zeros(6), 200.0 * np.ones(12)]; kd = np.r_[np.zeros(6), 2.0 * np.ones(12)]
    pt = gc.copy(); pt[:, 7::3] *= 1.5
    m = capi.Model(os.path.join(RSC, "anymal_c_like.urdf"))
    res = {}
    for on in (False, True):
        bt = capi.Batch(m, n)
        bt.set_params(gravity=(0.0, 0.0, 0.0), threshold=1e-6)
        if on:
            bt.set_self_collision(anymal_leg_pairs())
        bt.set_state(gc, gv); bt.set_pd_gains(kp, kd); bt.set_pd_target(pt, np.zeros((n, 18), np.float32))
        M = bt.mass_matrix().astype(np.float64)
        bt.integrate(1)
        res[on] = (M, bt.get_state()[1].astype(np.float64), bt.contacts()[0])
    M, v_on, ct = res[True]; v_off = res[False][1]
    # the same with the float32 oracle
    o = {on: SelfOracle(t, precision="f32", params=dict(gz=0.0, threshold=1e-6)) for on in (False, True)}
    o[True].set_self_collision(anymal_leg_pairs())
    ov = {}
    for on in (False, True):
        a, b = gc.astype(np.float64), gv.astype(np.float64)
        d = o[on].step(a, b, ptarget=pt.astype(np.float64), kp=kp, kd=kd, debug=True)
        ov[on] = (d["M"], b)

    def worst(M, von, voff):
        dv = von - voff
        imp = np.abs(np.einsum("eij,ej->ei", M, dv)).max(1)
        mom = np.abs(np.einsum("eij,ej->ei", M, von)).max(1)
        dP = np.abs(np.einsum("eij,ej->ei", M[:, :6], dv)).max(1)
        act = imp > 1e-3
        return act.sum(), (dP / (imp + mom))[act].max()
    na, wg = worst(M, v_on, v_off)
    nf, wf = worst(ov[True][0], ov[True][1], ov[False][1])
    print(f"environments with self impulses: GPU {na}, f32 oracle {nf}; momentum change relative: GPU {wg:.1e}, f32 oracle {wf:.1e}")
    assert na > n // 4 and (ct["pair_index"] < -1).any()
    assert wg < max(10 * wf, 1e-6)


# ---- 6: what the feature is for ------------------------------------------------------------------------------------------------

def test_knees_driven_together_stay_apart(capi, monkeypatch):
    """the front knees of the ANYmal-like robot driven into each other by PD (zero gravity, no terrain, joint stops off): with the knee
    pair enabled the spheres never cross and overlap by less than 4 cm -- ERP 0 keeps the depth reached in the first sub-step of contact,
    at most the approach speed times dt --; without it they pass through each other in every environment"""
    _env(monkeypatch)
    n = 64
    m = capi.Model(os.path.join(RSC, "anymal_c_like.urdf"))
    gc = np.tile(ANYMAL_GC0, (n, 1)); gc[:, 2] = 1.0
    gc[:, 7] += np.linspace(0.0, 0.2, n)
    pt = gc.copy(); pt[:, 7] = -1.4; pt[:, 10] = 1.4                       # hip abduction of both front legs far inwards
    sep = {}
    for on in (False, True):
        bt = capi.Batch(m, n)
        bt.set_params(gravity=(0.0, 0.0, 0.0), joint_limits=0)            # the hip abduction stops would keep the knees apart
        if on:
            bt.set_self_collision([(3, 7)])                                 # LF_SHANK/0 - RF_SHANK/0 (knee spheres, r = 0.055)
        bt.set_state(gc.astype(np.float32), np.zeros((n, 18), np.float32))
        bt.set_pd_gains(np.r_[np.zeros(6), 300.0 * np.ones(12)], np.r_[np.zeros(6), 10.0 * np.ones(12)])
        bt.set_pd_target(pt.astype(np.float32), np.zeros((n, 18), np.float32))
        worst, crossed = np.full(n, np.inf), np.zeros(n, bool)
        for _ in range(120):
            bt.integrate(4)
            R, p = bt.body_poses()
            lf, rf = p[:, 3], p[:, 6]                                       # knee sphere centres = the shank origins
            d = np.linalg.norm(lf - rf, axis=1)
            worst = np.minimum(worst, d)
            yb = np.einsum("eij,ej->ei", np.transpose(R[:, 0], (0, 2, 1)), lf - rf)[:, 1]   # LF left of RF in the base frame
            crossed |= yb < 0
        sep[on] = (worst, crossed)
    pen_on = 0.11 - sep[True][0]
    print(f"knee sphere distance min: pairs on {sep[True][0].min():.4f} m (penetration {pen_on.max():.4f}), off {sep[False][0].min():.4f} m, "
          f"crossed over without the pair in {int(sep[False][1].sum())} of {n}")
    assert pen_on.max() < 0.04 and not sep[True][1].any()
    assert sep[False][1].all()


# ---- 7: CTA sizes --------------------------------------------------------------------------------------------------------------

@pytest.mark.parametrize("name", list(CASES))
def test_self_collision_every_cta_size_bit_identical(capi, monkeypatch, name):
    """every CTA size that fits, two or more rounds ending on a partly filled CTA: bit-identical to the default pick"""
    import torch
    sms = torch.cuda.get_device_properties(0).multi_processor_count
    n = 2 * sms * 16 + 37
    ref, ran = None, []
    for wpc in (None, 28, 16, 14, 8, 4, 1):
        t, bt, _, _, gc, gv, cfg = _setup_wpc(capi, monkeypatch, name, n, wpc)
        if wpc is not None:
            if cfg["wpc"] != wpc:                           # this CTA does not fit in shared memory
                continue
            T = cfg["wpc"] * cfg["grid"]
            assert -(-n // T) >= 2 and n % T != 0
            ran.append(wpc)
        for _ in range(3):
            bt.integrate(4)
        out = _outputs(bt)
        if ref is None:
            ref = out
        else:
            _same(ref, out)
    print(f"{name}: CTA sizes run {ran}")
    assert len(ran) >= 4


def _setup_wpc(capi, monkeypatch, name, n, wpc):
    urdf, pairs, z = CASES[name]
    _env(monkeypatch, wpc=wpc)
    t, bt, o64, o32, _, _, _ = setup_batch(capi, urdf, n, 500, terrain="hm", tau_scale=0.0)
    bt.set_self_collision(pairs)
    cfg = launch_config(capi, bt)
    assert cfg["spec"] == SPEC_GENERIC
    gc, gv = _crossed(name, t, n, np.random.default_rng(501), z)
    bt.set_state(gc.astype(np.float32), gv.astype(np.float32))
    return t, bt, o64, o32, gc, gv, cfg


# ---- 8: refusals ---------------------------------------------------------------------------------------------------------------

def _call(capi, bt, pairs, mu=None):
    L = capi.lib()
    p = np.ascontiguousarray(np.asarray(pairs, np.int32).reshape(-1, 2))
    m = None if mu is None else np.ascontiguousarray(mu, np.float32)
    rc = L.rsb_batch_set_self_collision(bt.h, p.ctypes.data_as(ctypes.c_void_p), len(p), None if m is None else m.ctypes.data_as(ctypes.c_void_p))
    return rc, L.rsb_last_error().decode()


def test_self_collision_refusals_leave_batch_unchanged(capi, monkeypatch):
    """unsupported shapes (named in the message), two collision bodies of one body, more than 32 pairs and indices out of range are
    refused with the right code, and the batch runs exactly as before the call"""
    _env(monkeypatch)
    runs = []
    for refuse in (False, True):
        t, bt, _, _, _, _, _ = setup_batch(capi, "anymal_c_like.urdf", 256, 31, terrain="ground", tau_scale=20.0)
        bt.set_self_collision([(4, 8)])
        cfg = launch_config(capi, bt)
        if refuse:
            rc, msg = _call(capi, bt, [(4, 8), (0, 2)])                      # base box - thigh capsule
            assert rc == -4 and "box-capsule" in msg, msg
            rc, msg = _call(capi, bt, [(3, 4)])                              # both spheres of LF_SHANK
            assert rc == -1 and "same body" in msg, msg
            rc, msg = _call(capi, bt, [(4, 8)] * 33)
            assert rc == -1 and "at most 32" in msg, msg
            rc, msg = _call(capi, bt, [(4, 17)])
            assert rc == -1 and "out of range" in msg, msg
            rc, msg = _call(capi, bt, [(-1, 4)])
            assert rc == -1 and "out of range" in msg, msg
            assert launch_config(capi, bt) == cfg
        bt.integrate(4)
        runs.append(_outputs(bt))
    _same(runs[0], runs[1])
    # box-box and a cylinder
    _, bt, _, _, _, _, _ = setup_batch(capi, "atlas_like.urdf", 16, 1)
    rc, msg = _call(capi, bt, [(0, 1)])
    assert rc == -4 and "box-box" in msg, msg
    t = load_tables(MAX32)
    cyl = int(np.where(t["ctype"] == 3)[0][0]); sph = int(np.where((t["ctype"] == 0) & (t["cbody"] != t["cbody"][cyl]))[0][0])
    _, bt, _, _, _, _, _ = setup_batch(capi, MAX32, 16, 1)
    rc, msg = _call(capi, bt, [(sph, cyl)])
    assert rc == -4 and "cylinder" in msg, msg


# ---- 9: facade -----------------------------------------------------------------------------------------------------------------

def test_cpp_self_collision_example():
    """the raisim:: facade: setSelfCollisionPairs, getContacts() reporting isSelfCollision() with the other body, and
    ArticulatedSystem::ignoreCollisionBetween removing the knee pair (examples/self_collision.cpp)"""
    exe = os.path.join(ROOT, "examples", "self_collision")
    if not os.path.exists(exe):
        subprocess.check_call(["make", "-C", os.path.join(ROOT, "examples")])
    out = subprocess.run([exe, os.path.join(RSC, "anymal_c_like.urdf")], capture_output=True, text=True, timeout=120)
    print(out.stdout)
    assert out.returncode == 0, out.stdout + out.stderr
