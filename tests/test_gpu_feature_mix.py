"""Every per-environment feature at once, on every compiled variant of the step kernel (pytest -m gpu): each model of helpers.CASES and
the fixed-base pendulum, with and without an actuator network (AN) and actuation delays (DL), all other features on -- body inertia
rows, actuator rows (with -1, 0 and +inf entries), terrain friction rows, a three-map atlas on the quadrupeds and the hexapod, self
pairs on the generic ANYmal and Atlas, an external wrench in the first control step, per-body contact forces, frames and a height
scan -- against a float64 oracle per environment (tests/feature_mix_ref.py) with the float32 oracle's distance as the yardstick; then
bit-identity of the composed step under launch shapes, warps per CTA, row sources and setter order; then the gym task with all of it
on, terminations included, against the same composition."""
import os

import numpy as np
import pytest

from actuation_delay_ref import applied
from actuator_network_ref import random_layers, shift, torque
from body_inertia_ref import randomized, rows_of
from contact_force_ref import scatter_step
from feature_mix_ref import MixRef, dof_q
from frame_ref import batch_frame_kinematics, random_frames
from height_scan_ref import base_grid, sample_xy, surface_height
from helpers import _RSC, ANYMAL_GC0, CASES, FITS, PENDULUM_URDF, THRESH, _nominal, _pd, _state, fk_numpy, index_parity, launch_config
from oracle.urdf_tables import load_tables
from test_gpu_actuator_params import _random_rows
from oracle.gym_ref import observation
from test_gpu_contact_forces import _outputs, _same
from test_gpu_self_collision import ATLAS_PAIRS
from test_self_collision_oracle import anymal_leg_pairs

pytestmark = pytest.mark.gpu

SUB, STEPS, DT, H, L, W, DMAX = 4, 10, 0.0025, 3, 2, 32, 16
MODELS = dict(CASES, pendulum=(PENDULUM_URDF, False, (0, 1), None, None))
VARIANTS = {"none": (False, False), "AN": (True, False), "DL": (False, True), "AN+DL": (True, True)}
ATLAS = ("quad_feet", "anymal", "quad_prismatic", "quad_branched", "anymal_generic", "hexapod")     # the rest on flat ground
PAIRS = {"anymal_generic": anymal_leg_pairs(), "atlas_generic": ATLAS_PAIRS}
GEOM = (12.8, 9.6, 0.1, -0.2)
MU = 0.8            # the batch-level friction of collision body 0: the default material's, so the -1 entries of the rows stay at it
# one model per (spec, slots) pair
PER_INSTANCE = ("quad_feet", "anymal", "atlas", "quad_branched", "anymal_generic")
# the gym task's reset state: the quadruped drops and rolls, so that its base or thighs touch down within a few control steps and
# environments terminate, restart and terminate again inside a short run
GV_INIT = np.r_[0.0, 0.0, -2.0, 6.0, 0.0, 0.0, np.zeros(12)].astype(np.float32)


@pytest.fixture(scope="module")
def capi():
    import torch
    assert torch.cuda.is_available(), "GPU tests need a CUDA device"
    from raisimlib_b200 import capi as c
    return c


def _network_dofs(t):
    """every other joint dof and the last one: not contiguous, a count that is not a multiple of the kernel's group of 4, and dofs 32
    and 36 on the 37-dof model"""
    nbase = 6 if t["floating"] else 0
    d = list(range(nbase, t["nv"], 2))
    if d[-1] != t["nv"] - 1:
        d.append(t["nv"] - 1)
    if len(d) % 4 == 0:
        d = d[:-2] + d[-1:]
    return np.array(d)


def _inputs(name, variant, n, seed):
    """the seeded set-up of one run, shared by the batch and the reference"""
    urdf, generic, inst, _, _ = MODELS[name]
    path = os.path.join(_RSC, urdf) if urdf.endswith(".urdf") else urdf
    t = load_tables(path)
    rng = np.random.default_rng(seed)
    nv, nq = t["nv"], t["nq"]
    if t["floating"]:
        gc, gv = _state(name, t, n, rng)
        kp, kd, pt0 = _pd(t, n, _nominal(name, t), rng)
    else:
        gc = rng.uniform(-1, 1, (n, nq)).astype(np.float32).astype(np.float64)
        gv = (0.5 * rng.standard_normal((n, nv))).astype(np.float32).astype(np.float64)
        kp, kd = np.full(nv, 300.0), np.full(nv, 4.0)
        pt0 = rng.uniform(-1, 1, (n, nq)).astype(np.float32)
    nbase = 6 if t["floating"] else 0
    nj = nv - nbase
    cmds = []
    for _ in range(STEPS):
        pt = pt0.copy(); pt[:, nq - nj:] += rng.uniform(-0.25, 0.25, (n, nj)).astype(np.float32)
        vt = np.zeros((n, nv), np.float32); vt[:, nbase:] = rng.uniform(-1.0, 1.0, (n, nj))
        tau = np.zeros((n, nv), np.float32); tau[:, nbase:] = rng.uniform(-8.0, 8.0, (n, nj))
        cmds.append((pt, vt, tau))
    inertia = np.stack([rows_of(*randomized(t, rng)) for _ in range(n)])
    friction = rng.uniform(0.3, 1.2, (n, t["ncoll"])).astype(np.float32)
    friction[rng.random(friction.shape) < 0.2] = -1.0
    terrain = ("ground", 0.0)
    if name in ATLAS:
        hm = (0.1 * rng.uniform(-1, 1, (3, 49, 65))).astype(np.float32)
        terrain = ("atlas", GEOM, hm, (np.arange(n) * 7 % 3).astype(np.int32))
    an, dl = VARIANTS[variant]
    body = t["nb"] - 1
    wrench = (body, rng.uniform(-30, 30, (n, 3)).astype(np.float32), rng.uniform(-3, 3, (n, 3)).astype(np.float32),
              np.array([0.02, -0.01, 0.05], np.float32))
    return dict(name=name, t=t, path=path, generic=generic, inst=inst, n=n, gc=gc, gv=gv, kp=kp, kd=kd, cmds=cmds,
                rows=_random_rows(t, n, seed + 1), inertia=inertia, friction=friction, terrain=terrain, pairs=PAIRS.get(name),
                delay=(np.arange(n) % (DMAX + 1)).astype(np.int32) if dl else None,
                network=(_network_dofs(t), random_layers(np.random.default_rng(seed + 2), H, L, W), H) if an else None,
                wrench=wrench, bodies=list(range(min(t["nb"], 32))), frames=random_frames(rng, t["nb"], 5),
                scan=(np.zeros(25, np.int32), base_grid(5, 5, 0.6, 0.4)))


def _batch(capi, monkeypatch, x, wpc=None, delay=True, reverse=False, device=False):
    """the batch of _inputs x, every feature set; reverse: the setters in the opposite order, then the calls that rebuild the blob;
    device: the rows from device tensors"""
    import torch
    monkeypatch.setenv("RSB_FORCE_GENERIC", "1" if x["generic"] else "0")
    if wpc is None:
        monkeypatch.delenv("RSB_FORCE_WPC", raising=False)
    else:
        monkeypatch.setenv("RSB_FORCE_WPC", str(wpc))
    t, n = x["t"], x["n"]
    bt = capi.Batch(capi.Model(x["path"]), n)
    cuda = lambda a: torch.from_numpy(np.ascontiguousarray(a)).cuda()

    def terrain():
        if x["terrain"][0] == "ground":
            bt.set_ground(0.0)
        else:
            bt.set_heightmaps(*x["terrain"][1], x["terrain"][2], x["terrain"][3])
    setters = [lambda: bt.set_params(threshold=THRESH), terrain, lambda: bt.set_pd_gains(x["kp"], x["kd"]),
               lambda: bt.set_actuator_params_from(cuda(x["rows"])) if device else bt.set_actuator_params(x["rows"]),
               lambda: bt.set_body_inertia_from(cuda(x["inertia"])) if device else bt.set_body_inertia(x["inertia"]),
               lambda: bt.set_contact_friction_from(cuda(x["friction"])) if device else bt.set_contact_friction(x["friction"]),
               lambda: bt.set_contact_bodies(x["bodies"]), lambda: bt.set_frames(*x["frames"]), lambda: bt.set_height_scan(*x["scan"]),
               lambda: bt.set_collision_friction(0, MU) if t["ncoll"] else None]
    if x["pairs"] is not None:
        setters.append(lambda: bt.set_self_collision(x["pairs"]))
    if x["network"] is not None:
        setters.append(lambda: bt.set_actuator_network(*x["network"]))
    if x["delay"] is not None and delay:
        setters.append(lambda: bt.set_actuation_delay_from(cuda(x["delay"])) if device else bt.set_actuation_delay(x["delay"]))
    for s in (setters[::-1] if reverse else setters):
        s()
    if reverse:
        bt.set_params()
        if t["ncoll"]:
            bt.set_collision_friction(0, MU)
        bt.set_pd_gains(x["kp"], x["kd"]); terrain()
    bt.set_control_mode(capi.PD_PLUS_FEEDFORWARD_TORQUE)
    bt.set_state(x["gc"].astype(np.float32), x["gv"].astype(np.float32))
    return bt


def _command(bt, x, k):
    pt, vt, tau = x["cmds"][k]
    bt.set_pd_target(pt, vt)
    bt.set_generalized_force(tau)


def _wrench(bt, x):
    body, F, T, p = x["wrench"]
    bt.set_external_wrench(body, F, T, p)


def _run(bt, x, shape="first_one"):
    """the control steps of x; shape "first_one": the first control step as launches of 1 and SUB - 1 sub-steps (the outputs of the
    first sub-step are kept), "one": one launch of SUB per control step, "four": SUB launches of one.  Returns the outputs after every
    control step"""
    out = []
    for k in range(STEPS):
        _command(bt, x, k)
        launches = [1, SUB - 1] if (shape == "first_one" and k == 0) else [SUB] if shape in ("one", "first_one") else [1] * SUB
        for j, m in enumerate(launches):
            if k == 0:
                _wrench(bt, x)
            bt.integrate(m)
            if shape == "first_one" and k == 0 and j == 0:
                first = _outputs(bt)
                first["f"], first["s"] = bt.body_contact_forces()
                first["ct_rec"] = bt.contacts()[0]
                if x["network"] is not None:
                    first["hist"] = bt.actuator_history()
        o = _outputs(bt)
        if x["network"] is not None:
            o["hist"] = bt.actuator_history()
        if shape != "four":
            o["f"], o["s"] = bt.body_contact_forces()
        o["fpos"], o["frot"], o["flin"], o["fang"] = bt.frame_states()
        o["jac"] = bt.frame_jacobians()
        o["scan_h"], o["scan_xy"] = bt.height_scan()
        out.append(o)
    return (first, out) if shape == "first_one" else out


def _reference(x, precision):
    """the composition on the oracle of `precision`, one sub-step at a time: the debug outputs of the first sub-step and gv after it,
    gc and gv after every control step, solver statuses <= 1 in every sub-step, the self contacts seen"""
    t, n = x["t"], x["n"]
    ref = MixRef(t, n, precision=precision, params=dict(threshold=THRESH), kp=x["kp"], kd=x["kd"], rows=x["rows"],
                 inertia=x["inertia"].astype(np.float64), friction=x["friction"], terrain=x["terrain"], pairs=x["pairs"],
                 delay=x["delay"], network=x["network"])
    a, b = x["gc"].copy(), x["gv"].copy()
    body, F, T, p = x["wrench"]
    ext = (body, F.astype(np.float64), T.astype(np.float64), p.astype(np.float64))
    ok, selfc, first, states = np.ones(n, bool), 0, None, []
    for k in range(STEPS):
        for s in range(SUB):
            d = ref.substep(a, b, *x["cmds"][k], ext=ext if k == 0 else None)
            ok &= d["status"] <= 1
            live = np.arange(d["c_pt"].shape[1])[None, :] < d["ncontacts"][:, None]
            selfc += int((live & (d["c_pair"] < 0)).sum())
            if first is None:
                first, g1, v1 = d, a.copy(), b.copy()
        states.append((a.copy(), b.copy()))
    return dict(first=first, g1=g1, v1=v1, states=states, ok=ok, self_contacts=selfc, ref=ref)


def _sat(tau, lim):
    """actuators at their effort limit (an unlimited one never is)"""
    return np.isfinite(lim) & (np.abs(np.abs(tau) - lim) <= 1e-6 * lim)


# ---- a: every variant against the oracle -------------------------------------------------------------------------------------------

@pytest.mark.parametrize("variant", list(VARIANTS))
@pytest.mark.parametrize("name", list(MODELS))
def test_every_kernel_variant_matches_the_oracle(capi, monkeypatch, name, variant):
    n = 96
    x = _inputs(name, variant, n, seed=500 + 31 * list(MODELS).index(name) + list(VARIANTS).index(variant))
    t = x["t"]
    bt = _batch(capi, monkeypatch, x)
    cfg = launch_config(capi, bt)
    assert (cfg["spec"], cfg["slots"]) == x["inst"], f"{name}: runs {cfg}"
    first, got = _run(bt, x)
    r64, r32 = _reference(x, "f64"), _reference(x, "f32")
    d, d32 = r64["first"], r32["first"]
    lim = r64["ref"].lim
    # the variant took effect: the network torque of the first sub-step and its history; the delays move the trajectory
    if x["network"] is not None:
        dofs, layers, _ = x["network"]
        q = dof_q(t)[dofs]
        pt, vt, tau = x["cmds"][0]
        g0, v0 = x["gc"].astype(np.float32), x["gv"].astype(np.float32)
        e, v = pt[:, q] - g0[:, q], v0[:, dofs]
        want = torque(layers, e, v, np.zeros((n, len(dofs), 2, H - 1)), tau[:, dofs], lim[:, dofs])
        err = np.abs(first["tau"][:, dofs] - want) / (1.0 + np.abs(want))
        assert err.max() <= 1e-4 and np.abs(want).max() > 5.0, err.max()
        assert first["hist"].tobytes() == shift(e, v, np.zeros((n, len(dofs), 2, H - 1), np.float32)).tobytes()
        assert np.abs(d["tau_net"] - want).max() < 1e-3 * (1 + np.abs(want).max())
    if x["delay"] is not None:
        plain = _batch(capi, monkeypatch, x, delay=False)
        _, gp = _run(plain, x)
        dl = x["delay"] > 0
        assert (gp[-1]["gc"][dl] != got[-1]["gc"][dl]).any(1).all()
    # the edges: contacts, joint-limit rows, saturated actuators, self contacts
    sat_ref = _sat(d["tau_applied"], lim)[:, 6 if t["floating"] else 0:]
    assert sat_ref.any()
    if t["npts"]:
        assert first["cnt"].sum() > n // 4
    if (np.abs(t["jlimit"][1:]) < 1e29).any():
        assert d["nlimits"].sum() > 0
    if x["pairs"] is not None:
        assert r64["self_contacts"] > 0
    # contact lists of the first sub-step, the saturation switch, gv after it
    hard = index_parity(first["pts"], first["cnt"], d32, f"{name} {variant}")
    assert hard.sum() <= (0 if x["terrain"][0] == "ground" else 1), f"contact lists differ in envs {np.where(hard)[0][:10]}"
    sat_gpu = _sat(first["tau"].astype(np.float64), lim)[:, 6 if t["floating"] else 0:]
    assert (sat_gpu == sat_ref).mean() > 0.999, f"{int((sat_gpu != sat_ref).sum())} actuators switched differently"
    conv = (first["pts"] == d["c_pt"]).all(1) & (first["st"] == 0) & (d["status"] == 0)
    v64, v32 = r64["v1"], r32["v1"]
    ev, e32 = np.abs(first["gv"] - v64)[conv], np.abs(v32 - v64)[conv]
    scale_v = 1.0 + np.abs(v64[conv])
    assert conv.mean() > 0.8
    assert np.median(ev.max(1)) < max(2e-5, 3 * np.median(e32.max(1)))
    assert np.max(ev / scale_v) < max(5e-3, 3 * np.max(e32 / scale_v))
    eq = np.abs(first["gc"] - r64["g1"])[conv]
    assert eq.max() < 5e-3 * DT * (1.0 + np.abs(v64[conv]).max()) + 2e-6
    # Signorini and Coulomb on the GPU's own contact records, each contact with its environment's friction row
    ct, cnt = first["ct_rec"], first["cnt"]
    K = ct.shape[1]
    on = np.arange(K)[None, :] < cnt[:, None]
    pt_ = first["pts"][:, :K]
    coll = np.where((pt_ >= 0) & (pt_ < t["npts"]), np.asarray(t["pt_coll"])[np.clip(pt_, 0, max(t["npts"] - 1, 0))] if t["npts"] else -1, -1)
    row = np.take_along_axis(x["friction"], np.clip(coll, 0, None), 1) if t["ncoll"] else np.full(coll.shape, -1.0)
    mu = np.where((coll >= 0) & (row >= 0), row, MU)
    ln = np.einsum("ekj,ekj->ek", ct["impulse"], ct["normal"])
    lt = np.linalg.norm(ct["impulse"] - ln[:, :, None] * ct["normal"], axis=2)
    assert (ln[on] >= -1e-6).all() and (lt[on] <= mu[on] * ln[on] + 1e-4 * (1 + ln[on])).all()
    # contact forces per body in the first sub-step
    (f64, h64), (f32, _) = scatter_step(d, x["bodies"]), scatter_step(d32, x["bodies"])
    assert (first["s"][conv] == h64[conv]).all()
    fs = max(1.0, np.abs(d["c_lambda"][:, :, 2]).max()) / DT
    ef, ef32 = np.abs(first["f"] - f64 / DT)[conv].max((1, 2)), np.abs(f32 - f64)[conv].max((1, 2)) / DT
    assert np.median(ef) < max(1e-4 * fs, 3 * np.median(ef32)) and np.quantile(ef, 0.99) < max(1e-4 * fs, 5 * np.quantile(ef32, 0.99))
    # gc after all control steps
    ok = r64["ok"] & r32["ok"] & np.logical_and.reduce([o["st"] <= 1 for o in got])
    # The bounds of helpers.step_and_trajectory, taken over 40 sub-steps instead of 10 and with a network on up to 15 dofs: the
    # absolute floors stay, but the float32 oracle's own distance from the float64 one (median 2.5e-4 on the humanoid with a network,
    # against the 2e-5 floor) is the yardstick, as in tests/test_gpu_actuator_network.py.  Flips: on the rough atlas index parity
    # allows a contact list to differ on a tie, and a robot whose contact set changed follows another trajectory from there; as in
    # step_and_trajectory the worst n // 25 environments leave the quantiles there (none on flat ground).  The sample is the
    # environments whose solves end at status <= 1 in every sub-step on all three sides: self contacts of the humanoid stall the
    # solve of about a quarter of them somewhere in 40 sub-steps, hence 0.7 rather than the one-step share of 0.8.
    flips = n // 25 if x["terrain"][0] == "atlas" else 0
    gN, a64, a32 = got[-1]["gc"], r64["states"][-1][0], r32["states"][-1][0]
    eg, eg32 = np.sort(np.abs(gN - a64).max(1)[ok])[:int(ok.sum()) - flips], np.abs(a32 - a64).max(1)[ok]
    print(f"| {name:15s} | spec {cfg['spec']} | slots {cfg['slots']} | AN {int(x['network'] is not None)} | DL {int(x['delay'] is not None)} | "
          f"1 sub-step gv err median {np.median(ev.max(1)):.1e} (f32 {np.median(e32.max(1)):.1e}) | {STEPS * SUB} sub-steps gc err median "
          f"{np.median(eg):.1e} p90 {np.quantile(eg, .9):.1e} max {eg.max():.1e} (f32 median {np.median(eg32):.1e} p90 "
          f"{np.quantile(eg32, .9):.1e} max {eg32.max():.1e}) | converged {100 * ok.mean():.0f} % | saturated {int(sat_ref.sum())} | self contacts {r64['self_contacts']} |")
    assert ok.mean() > 0.7 and np.isfinite(gN).all()
    assert np.median(eg) < max(2e-5, 5 * np.median(eg32))
    assert np.quantile(eg, 0.9) < max(1e-4, 5 * np.quantile(eg32, 0.9))
    assert np.quantile(eg, 0.99) < max(5e-3, 5 * np.quantile(eg32, 0.99))
    # frames and height scan at the GPU's final state: frame_ref on float64 kinematics, and the surface of each environment's own map
    g, v_ = got[-1]["gc"].astype(np.float64), got[-1]["gv"].astype(np.float64)
    body, pos, rot = x["frames"]
    fx, fR, fl, fa, fJ = batch_frame_kinematics(t, g, v_, body, pos, rot)
    px, pR, pl, pa, pJ = (got[-1][k_] for k_ in ("fpos", "frot", "flin", "fang", "jac"))
    assert np.abs(px - fx).max() < 1e-4 and np.abs(pR - fR).max() < 1e-4
    assert np.abs(pl - fl).max() < 1e-3 * (1 + np.abs(fl).max()) and np.abs(pa - fa).max() < 1e-3 * (1 + np.abs(fa).max())
    assert np.abs(pJ - fJ).max() < 1e-4 * (1 + np.abs(fJ).max())
    hs, hxy = got[-1]["scan_h"], got[-1]["scan_xy"]
    poses = [fk_numpy(t, g[e]) for e in range(n)]
    want_xy = sample_xy(np.stack([q_[0] for q_ in poses]), np.stack([q_[1] for q_ in poses]), *x["scan"])
    assert np.abs(hxy - want_xy).max() < 1e-4
    if x["terrain"][0] == "atlas":
        hm, emap = x["terrain"][2], x["terrain"][3]
        want_h = np.stack([surface_height(hm[emap[e]], *GEOM, hxy[e, :, 0], hxy[e, :, 1]) for e in range(n)])
    else:
        want_h = np.zeros_like(hs, np.float64)
    assert np.abs(hs - want_h).max() < 1e-5
    # past the delay counter's wrap, the network still reads the applied target: one more sub-step, its history bit for bit
    if x["network"] is not None:
        g, v_ = bt.get_state()
        h0 = bt.actuator_history()
        bt.integrate(1)
        s = STEPS * SUB
        delay = x["delay"] if x["delay"] is not None else np.zeros(n, np.int32)
        k = np.minimum([applied(np.arange(s + 1), int(de))[-1] // SUB for de in delay], STEPS - 1)
        pt_app = np.stack([x["cmds"][k[j]][0][j] for j in range(n)])
        assert bt.actuator_history().tobytes() == shift(pt_app[:, q] - g[:, q], v_[:, dofs], h0).tobytes()


# ---- b: invariance with everything on ------------------------------------------------------------------------------------------------

def _control_steps(bt, x):
    """control_step (targets in, observation out, one launch) instead of set_pd_target + integrate + observe; the outputs of _run"""
    out = []
    obs = np.empty((x["n"], bt.ob_dim()), np.float32)
    for k in range(STEPS):
        pt, vt, tau = x["cmds"][k]
        bt.set_generalized_force(tau)
        if k == 0:
            _wrench(bt, x)
        bt.control_step(pt, SUB, obs, vtarget=vt)
        o = _outputs(bt)
        o["hist"] = bt.actuator_history()
        o["f"], o["s"] = bt.body_contact_forces()
        o["fpos"], o["frot"], o["flin"], o["fang"] = bt.frame_states()
        o["jac"] = bt.frame_jacobians()
        o["scan_h"], o["scan_xy"] = bt.height_scan()
        assert obs.tobytes() == o["obs"].tobytes()
        out.append(o)
    return out


@pytest.mark.parametrize("name", PER_INSTANCE)
def test_everything_on_gives_the_same_bits_under_every_launch_and_set_up(capi, monkeypatch, name):
    """network and delays on with every other feature: each warps-per-CTA choice, one launch of 4 sub-steps against 4 launches of 1,
    control_step, rows from device tensors, and the setters in reverse order followed by the calls that rebuild the model blob.  300
    environments: several rounds of CTAs at the small warps-per-CTA choices, the last one partly filled"""
    n = 300
    x = _inputs(name, "AN+DL", n, seed=900 + list(MODELS).index(name))
    ref = _run(_batch(capi, monkeypatch, x), x, "one")
    runs, rounds = {}, []
    for w in FITS[name]:
        bt = _batch(capi, monkeypatch, x, wpc=w)
        cfg = launch_config(capi, bt)
        if cfg["wpc"] != w:         # the self pairs' larger workspace: this CTA does not fit, the launch keeps its own choice
            continue
        rounds.append((w, -(-n // (cfg["wpc"] * cfg["grid"]))))
        runs[f"wpc {w}"] = _run(bt, x, "one")
    print(f"{name}: (warps per CTA, CTA rounds) taken {rounds} of {FITS[name]}")
    assert len(rounds) >= 3 and max(r for _, r in rounds) > 1
    runs["control_step"] = _control_steps(_batch(capi, monkeypatch, x), x)
    runs["device rows"] = _run(_batch(capi, monkeypatch, x, device=True), x, "one")
    runs["reverse order"] = _run(_batch(capi, monkeypatch, x, reverse=True), x, "one")
    if name == "anymal":
        for pair in ("0", "1"):
            for barrier in ("0", "1"):
                monkeypatch.setenv("RSB_PAIR_STAGE_A", pair); monkeypatch.setenv("RSB_SUBSTEP_BARRIER", barrier)
                runs[f"pair stage A {pair} barrier {barrier}"] = _run(_batch(capi, monkeypatch, x), x, "one")
        monkeypatch.delenv("RSB_PAIR_STAGE_A"); monkeypatch.delenv("RSB_SUBSTEP_BARRIER")
    four = _run(_batch(capi, monkeypatch, x), x, "four")
    assert sum(int(o["cnt"].sum()) for o in ref) > n and np.abs(ref[-1]["hist"]).max() > 0
    for what, out in runs.items():
        for k in range(STEPS):
            _same(ref[k], out[k], f"{name} {what}, control step {k}: ")
    for k in range(STEPS):
        _same({key: v for key, v in ref[k].items() if key not in ("f", "s")}, four[k], f"{name} four launches, control step {k}: ")


# ---- c: the gym task with everything on --------------------------------------------------------------------------------------------

class _MixOracle:
    """the oracle GymRef drives, made of the per-environment composition: step() runs its sub-steps one at a time, with no feed-forward
    torque, and returns the debug outputs of the last one"""

    def __init__(self, mix):
        self.mix = mix

    def reset_warm_start(self, n):
        for o in self.mix.oracles:
            o.reset_warm_start(1)

    def step(self, gc, gv, n_steps, ptarget, vtarget, kp, kd, debug):
        for _ in range(n_steps):
            d = self.mix.substep(gc, gv, ptarget, vtarget, np.zeros_like(gv))
        return d


@pytest.mark.parametrize("name", ["anymal", "anymal_generic"])
def test_gym_task_with_everything_on_matches_the_composition(capi, monkeypatch, name):
    """20 gym steps with the network, delays 0 .. 16 and every row on: rewards, done flags and observations against oracle.gym_ref.GymRef
    around the per-environment composition, with the bounds of test_gpu_parity.test_gym_task_matches_numpy_restatement.  A termination
    zeroes that environment's network history and empties its command history (the composition restarts its delay there), and keeps
    every row (the composition keeps them)"""
    from oracle.gym_ref import GymRef
    n, steps = 96, 20
    x = _inputs(name, "AN+DL", n, seed=1300 + len(name))
    t = x["t"]
    bt = _batch(capi, monkeypatch, x)
    gc_init = _nominal(name, t).astype(np.float32)
    feet = [3, 6, 9, 12]
    bt.set_generalized_force(np.zeros((n, t["nv"]), np.float32))
    bt.set_pd_target(np.tile(gc_init, (n, 1)), np.zeros((n, t["nv"]), np.float32))
    bt.gym_configure(gc_init, GV_INIT, gc_init[7:], 0.6 * np.ones(12), feet)
    bt.gym_reset()
    mixes = [MixRef(t, n, precision=p, params=dict(threshold=THRESH), kp=x["kp"], kd=x["kd"], rows=x["rows"],
                    inertia=x["inertia"].astype(np.float64), friction=x["friction"], terrain=x["terrain"], pairs=x["pairs"],
                    delay=x["delay"], network=x["network"]) for p in ("f64", "f32")]
    refs = [GymRef(_MixOracle(mix), gc_init, GV_INIT, gc_init[7:], (0.6 * np.ones(12)).astype(np.float32), feet, x["kp"], x["kd"])
            for mix in mixes]
    for ref in refs:
        ref.reset(n)
    rng = np.random.default_rng(1400)
    base = rng.normal(0, 1.5, (n, 12))
    obs, rew, done = np.empty((n, bt.ob_dim()), np.float32), np.empty(n, np.float32), np.empty(n, np.uint8)
    agree, n_done, restarted = np.ones(n, bool), 0, 0
    for k in range(steps):
        act = (base + rng.normal(0, 0.3, (n, 12))).astype(np.float32)
        bt.gym_step(act, SUB, obs, rew, done)
        out = [ref.step(act.astype(np.float64), SUB) for ref in refs]
        for mix, (_, _, d_, _) in zip(mixes, out):
            mix.reset_network_history(np.nonzero(d_)[0])
            mix.empty_delay_history(np.nonzero(d_)[0])
        (o_ref, r_ref, d_ref, _), (o32, r32, d32, _) = out
        agree &= done.astype(bool) == d_ref
        n_done += int(d_ref.sum())
        restarted += int((agree & d_ref).sum()) if k < steps - 1 else 0
        a = agree & (d32 == d_ref)
        assert a.mean() > 0.9, f"gym step {k}"
        # The 5e-3 bound of the plain gym test.  Robots that land on their backs and sides make the trajectories of a tenth or more of
        # the environments sensitive to rounding: the float32 composition itself leaves 5e-3 of the float64 one in that many.  So
        # the kernel may leave it in at most twice as many environments as the float32 composition does, plus 5 %, and the typical
        # environment stays within the plain test's reach.
        eo, er = np.abs(obs[a] - o_ref[a]).max(1), np.abs(rew[a] - r_ref[a])
        eo32, er32 = np.abs(o32[a] - o_ref[a]).max(1), np.abs(r32[a] - r_ref[a])
        rs = 5e-3 * (1 + np.abs(r_ref[a]).max())
        assert (eo > 5e-3).mean() <= 2 * (eo32 > 5e-3).mean() + 0.05, (k, (eo > 5e-3).mean(), (eo32 > 5e-3).mean())
        assert (er > rs).mean() <= 2 * (er32 > rs).mean() + 0.05, (k, (er > rs).mean(), (er32 > rs).mean())
        assert np.median(eo) < max(1e-4, 5 * np.median(eo32)) and np.median(er) < max(1e-4 * rs, 5 * np.median(er32))
        h = bt.actuator_history()
        assert not h[done == 1].any(), f"gym step {k}: a terminated environment kept its network history"
        assert (np.abs(h[done == 0]).reshape(int((done == 0).sum()), -1).max(1) > 0).all()
    print(f"{name}: {n_done} terminations over {steps} gym steps, {restarted} of them compared after the restart, "
          f"{100 * agree.mean():.0f} % of the environments in lockstep to the end")
    assert restarted > 5
