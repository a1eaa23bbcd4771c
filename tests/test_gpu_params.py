"""The step kernel against the oracle with every solver and integrator parameter of rsb_params off its default (run on an H100:
pytest -m gpu), on every compiled instance (CASES of tests/helpers.py, each asserted through rsb_internal_launch_config).

The integrator runs at other time steps and gravities, with the ERP / restitution row bias at the ends of the time-step range and
with joint limits off; the solver runs a fixed number of sweeps (its iterates, not only its fixed point, against the oracle's), other
relaxation schedules, and exits that depend on integer sweep counts alone, so the status and sweep count of every solve are compared
exactly.  Tolerances are the float32-oracle envelope of tests/test_gpu_instances.py: the kernel may be at most about 3x (one step) or
5x (10 steps) further from the float64 oracle than the float32 build of the oracle is.  rsb_batch_set_params itself: what is set is
what is read back and what the next launch runs, and a refused call changes nothing."""
import ctypes

import numpy as np
import pytest

from contact_force_ref import world_impulses
from helpers import CASES, THRESH, ROW_BIAS, _batch, launch_config, step_and_trajectory
from test_gpu_contact_forces import _scatter_records

pytestmark = pytest.mark.gpu

TERRAINS = ("ground", "hm")
# rsb_params_default, with the solver threshold the parity tests run on both sides (THRESH); gx, gy, gz are the gravity vector
DEFAULTS = dict(dt=0.0025, gx=0.0, gy=0.0, gz=-9.81, erp=0.0, alpha_init=1.0, alpha_min=1.0, alpha_decay=1.0, max_iter=150, threshold=THRESH,
                mu=0.8, restitution=0.0, rest_threshold=0.01, stall_window=8, stall_ratio=0.5, joint_limits=1, accel_m=2, accel_start=6,
                stall_reg=0.02)
CONVERGED, COMPLIANT, STALLED, MAXITER = 0, 1, 2, 3        # RSB_SOLVER_*


@pytest.fixture(scope="module")
def capi():
    import torch
    assert torch.cuda.is_available(), "GPU tests need a CUDA device"
    from raisimlib_b200 import capi as c
    return c


def _seed(name, terrain, salt):
    return 5000 + 31 * len(name) + 7 * (terrain == "hm") + salt


def _compare(capi, monkeypatch, name, terrain, salt, params, **kw):
    """step_and_trajectory away from the defaults: stiffer friction, full restitution, large steps and other gravities leave more solves
    on the compliant set or stalled on one side (at least 60 % converge on both: the ERP bias of a 1 ms step on the 32-body star sunk in
    the rough map stalls a third of its solves), and on the rough map up to 10 of the 256 robots may
    take a contact set one step apart from the oracle's, one per step as index parity allows"""
    return step_and_trajectory(capi, monkeypatch, name, terrain, _seed(name, terrain, salt), params=params, converged=0.6,
                               flips=10 if terrain == "hm" else 0, **kw)


CASE_TERRAINS = [pytest.param(name, terrain, id=f"{name}-{terrain}") for name in CASES for terrain in TERRAINS]


# ---- 1: integrator ------------------------------------------------------------------------------------------------------------------

@pytest.mark.parametrize("dt", [0.001, 0.005, 0.01])
@pytest.mark.parametrize("name,terrain", CASE_TERRAINS)
def test_time_step(capi, monkeypatch, name, terrain, dt):
    """one step and 10 steps at another dt: stages C and E, the PD law's implicit terms, the effort-limit threshold
    tau_max (1 + (dt kd + dt^2 kp) / M_dd) and the integration all take dt from the parameters"""
    _compare(capi, monkeypatch, name, terrain, 1, dict(dt=dt))


@pytest.mark.parametrize("dt", [0.001, 0.01])
@pytest.mark.parametrize("name,terrain", CASE_TERRAINS)
def test_row_bias_time_step(capi, monkeypatch, name, terrain, dt):
    """ERP enters as erp * depth / dt and erp * violation / dt: the row bias at both ends of the time-step range"""
    _compare(capi, monkeypatch, name, terrain, 2, dict(ROW_BIAS, dt=dt), near_threshold="exclude")


@pytest.mark.parametrize("gravity", [(0.0, 0.0, 0.0), (3.0, -2.0, -9.81), (0.0, 0.0, -1.62)], ids=["zero", "tilted", "moon"])
@pytest.mark.parametrize("name,terrain", CASE_TERRAINS)
def test_gravity(capi, monkeypatch, name, terrain, gravity):
    """stage A's base acceleration is minus the gravity vector on every instance, the quadruped's paired stage A included"""
    _compare(capi, monkeypatch, name, terrain, 3, dict(gx=gravity[0], gy=gravity[1], gz=gravity[2]))


@pytest.mark.parametrize("terrain", TERRAINS)
@pytest.mark.parametrize("name", ["quad_feet", "anymal", "quad_prismatic", "atlas"])
def test_joint_limits_off(capi, monkeypatch, name, terrain):
    """joint_limits = 0 on the quadruped and humanoid instances: no limit rows although joints start past their stops"""
    _compare(capi, monkeypatch, name, terrain, 4, dict(joint_limits=0))


# ---- 2-4: the solver's iterates, relaxation and exits -----------------------------------------------------------------------------

class _Rig:
    """one batch and both oracles on the same start state; run() takes one step from it with a complete parameter set on every side"""

    def __init__(self, capi, monkeypatch, name, terrain, seed, n=256):
        self.t, self.bt, self.o64, self.o32, self.gc, self.gv, self.kp, self.kd, self.pt, self.cfg = _batch(capi, monkeypatch, name, n, terrain, seed)
        self.name, self.terrain, self.n = name, terrain, n

    def run(self, **over):
        prm = dict(DEFAULTS, **over)
        self.bt.set_params(gravity=(prm["gx"], prm["gy"], prm["gz"]), **{k: v for k, v in prm.items() if k not in ("gx", "gy", "gz")})
        for o in (self.o64, self.o32):
            o.set_params(**prm)
        self.bt.set_state(self.gc.astype(np.float32), self.gv.astype(np.float32))
        self.bt.integrate(1)
        _, v1 = self.bt.get_state(); ct, cnt = self.bt.contacts()
        r = dict(v1=v1, imp=ct["impulse"].astype(np.float64), cnt=cnt, pts=self.bt.contact_points(), st=self.bt.solver_status(),
                 it=self.bt.solver_iterations(), resid=self.bt.solver_residual().astype(np.float64), prm=prm)
        kw = dict(ptarget=self.pt.astype(np.float64), vtarget=np.zeros((self.n, self.t["nv"])), kp=self.kp, kd=self.kd, debug=True)
        r["b64"], r["b32"] = self.gv.copy(), self.gv.copy()
        r["d"] = self.o64.step(self.gc.copy(), r["b64"], **kw)
        r["d32"] = self.o32.step(self.gc.copy(), r["b32"], **kw)
        d = r["d"]
        r["rows"] = 3 * d["ncontacts"] + d["nlimits"]
        r["same"] = (r["pts"] == d["c_pt"]).all(1) & (cnt == d["ncontacts"])
        r["same32"] = r["same"] & (r["d32"]["c_pt"] == d["c_pt"]).all(1) & (r["d32"]["nlimits"] == d["nlimits"])
        return r


def _no_rows_report_nothing(r):
    """environments without contacts and limit rows run no sweep and report converged, on both sides"""
    none = r["same"] & (r["rows"] == 0)
    assert (r["it"][none] == 0).all() and (r["st"][none] == CONVERGED).all()
    assert (r["d"]["iters"][none] == 0).all() and (r["d"]["status"][none] == CONVERGED).all()


def _iterate_errors(r, sel):
    """kernel and float32-oracle distances from the float64 oracle after one step, over the environments sel: gv+ and the world
    contact impulses"""
    sel = sel & r["same32"]
    imp64, imp32 = world_impulses(r["d"]), world_impulses(r["d32"])
    live = sel[:, None] & (r["d"]["c_pt"] >= 0)
    ei = np.abs(r["imp"] - imp64).max(2)[live]; ei32 = np.abs(imp32 - imp64).max(2)[live]
    scale_i = max(1.0, np.abs(imp64[live]).max()) if live.any() else 1.0
    ev, ev32 = np.abs(r["v1"] - r["b64"])[sel], np.abs(r["b32"] - r["b64"])[sel]
    return sel, ei, ei32, scale_i, ev, ev32, 1.0 + np.abs(r["b64"][sel])


def _within_envelope(r, sel, label, share=0.5, tail=False):
    """kernel within the float32-oracle envelope on every environment of sel: median and largest gv+ error over its scale, and the
    99th percentile of the contact impulse errors.  tail: after an Anderson step the largest errors are compared as a count instead --
    the environments with a gv+ or impulse error outside 3x the float32 oracle's 90th percentile (or the floor), kernel against float32
    oracle"""
    sel, ei, ei32, scale_i, ev, ev32, scale_v = _iterate_errors(r, sel)
    assert sel.sum() > share * r["same"].size, f"{label}: only {sel.sum()} environments compared"
    live = r["d"]["c_pt"][sel] >= 0
    env_of = np.broadcast_to(np.arange(sel.sum())[:, None], live.shape)[live]      # environment of each entry of ei
    rv, rv32 = (ev / scale_v).max(1), (ev32 / scale_v).max(1)
    p99, p99_32 = (np.quantile(ei, 0.99), np.quantile(ei32, 0.99)) if ei.size else (0.0, 0.0)
    line = (f"     {label:34s} | envs {sel.sum():3d} | gv err median {np.median(ev.max(1)):.1e} (f32 {np.median(ev32.max(1)):.1e}) max/scale "
            f"{rv.max():.1e} (f32 {rv32.max():.1e}) | impulse p99 {p99:.1e} (f32 {p99_32:.1e}, scale {scale_i:.1f})")
    assert np.median(ev.max(1)) < max(2e-5, 3 * np.median(ev32.max(1))), label
    if not tail:
        print(line)
        assert rv.max() < max(5e-3, 3 * rv32.max()), label
        assert p99 < max(1e-4 * scale_i, 3 * p99_32), label
        return
    ev_env = max(5e-3, 3 * np.quantile(rv32, 0.9))
    ei_env = max(1e-4 * scale_i, 3 * np.quantile(ei32, 0.9)) if ei.size else 0.0
    out, out32 = int((rv > ev_env).sum()), int((rv32 > ev_env).sum())
    outi, outi32 = len(np.unique(env_of[ei > ei_env])), len(np.unique(env_of[ei32 > ei_env]))
    print(line + f" | beyond the envelope: gv {out} (f32 {out32}), impulses {outi} (f32 {outi32})")
    assert out <= 2 * out32 + 3 and outi <= 2 * outi32 + 3, label


def _fixed_sweeps(r, k, label):
    """threshold 0 and no stagnation check: every solve with a row runs exactly k sweeps and ends MAXITER, on both sides.  Once an
    Anderson step has been taken before the last sweep (k > accel_start), the extrapolation has solved a least-squares problem on
    residual differences near rounding: it amplifies float32 rounding in a few environments, on the float32 oracle as on the kernel
    (each prints how many of its environments lie beyond the envelope), so there the tail is compared as a count."""
    has = r["same"] & (r["rows"] > 0)
    assert r["same"].mean() > 0.95 and has.mean() > 0.5
    assert (r["d"]["iters"][has] == k).all() and (r["d"]["status"][has] == MAXITER).all()
    assert (r["it"][has] == k).all(), f"{label}: sweeps {np.unique(r['it'][has]).tolist()}, expected {k}"
    assert (r["st"][has] == MAXITER).all(), f"{label}: statuses {np.bincount(r['st'][has], minlength=4).tolist()}"
    _no_rows_report_nothing(r)
    _within_envelope(r, has, label, tail=r["prm"]["accel_m"] > 0 and k > r["prm"]["accel_start"])


FIXED = dict(threshold=0.0, stall_window=0)


@pytest.mark.parametrize("name,terrain", CASE_TERRAINS)
def test_solver_iterates_at_fixed_sweep_counts(capi, monkeypatch, name, terrain):
    """k sweeps exactly, plain and accelerated: the impulses and gv+ after k sweeps against the oracle's after k sweeps.  k runs
    through the first extrapolations (accel_start 3 and 6) and k = accel_start, whose last sweep is never extrapolated"""
    rig = _Rig(capi, monkeypatch, name, terrain, _seed(name, terrain, 5))
    print(f"\n{name} {terrain}: {launch_config(capi, rig.bt)}")
    for m, start in ((0, 6), (2, 3), (2, 6)):
        for k in (1, 2, 3, 4, 5, 6, 7, 8, 12):
            r = rig.run(max_iter=k, accel_m=m, accel_start=start, **FIXED)
            _fixed_sweeps(r, k, f"accel_m {m} accel_start {start} k {k:2d}")


SCHEDULES = [(0.5, 0.5, 1.0), (1.0, 0.4, 0.9), (1.3, 1.3, 1.0)]


@pytest.mark.parametrize("name,terrain", CASE_TERRAINS)
def test_relaxation_schedule(capi, monkeypatch, name, terrain):
    """alpha_init, alpha_min, alpha_decay: under- and over-relaxation and a decaying factor, after 5 sweeps and run to convergence"""
    rig = _Rig(capi, monkeypatch, name, terrain, _seed(name, terrain, 6))
    print(f"\n{name} {terrain}: {launch_config(capi, rig.bt)}")
    for a0, amin, adec in SCHEDULES:
        sched = dict(alpha_init=a0, alpha_min=amin, alpha_decay=adec)
        _fixed_sweeps(rig.run(max_iter=5, **FIXED, **sched), 5, f"alpha {a0} / {amin} / {adec}, 5 sweeps")
        r = rig.run(**sched)
        st, s64 = r["st"][r["same"]], r["d"]["status"][r["same"]]
        print(f"     alpha {a0} / {amin} / {adec} to convergence: status gpu {np.bincount(st, minlength=4).tolist()} oracle "
              f"{np.bincount(s64, minlength=4).tolist()}")
        assert (st == s64).mean() > 0.9
        _no_rows_report_nothing(r)
        conv = r["same"] & (r["st"] == CONVERGED) & (r["d"]["status"] == CONVERGED)
        _within_envelope(r, conv, f"alpha {a0} / {amin} / {adec}, converged", share=0.25)


def _predicted_exit(resid, checkpoints, reg, max_iter, n):
    """the (status, sweeps) that threshold 0 and stall_ratio 0 imply, from the largest update at each checkpoint 2w, 3w, ... <= max_iter
    (resid[c]): every checkpoint whose update is not 0 fails -- the first turns the set compliant when reg > 0, the next (or with reg 0
    the first) ends the solve STALLED there; an update of exactly 0 passes"""
    st, it = np.full(n, MAXITER), np.full(n, max_iter)
    done, regd = np.zeros(n, bool), np.zeros(n, bool)
    for c in checkpoints:
        fail = ~done & (resid[c] > 0)
        stall = fail & regd if reg > 0 else fail
        regd |= fail & ~stall
        st[stall], it[stall] = STALLED, c
        done |= stall
    return st, it


def _exits(rig, w, reg, max_iter, label):
    """stall_ratio 0, threshold 0: one run to max_iter, and one run stopped at each checkpoint c >= 2w (max_iter = c) whose last update
    is the largest update at checkpoint c of the full run -- the sweeps before it are the same, and the Anderson step that a stop
    leaves out comes after the update is measured.  Every solve with a row must end as its own checkpoint updates dictate, on the
    kernel and on both oracle builds; and the kernel's (status, sweeps) must equal the float64 oracle's wherever the two agree on
    which checkpoint updates are exactly 0.  Where they do not, one side reached an exact float32 fixed point: the other side's update
    at that checkpoint must be at rounding level, and such environments must be few."""
    base = dict(threshold=0.0, stall_ratio=0.0, stall_window=w, stall_reg=reg)
    checkpoints = list(range(2 * w, max_iter + 1, w))
    full = rig.run(max_iter=max_iter, **base)
    has = full["same"] & (full["rows"] > 0)
    rk, r64, r32 = {}, {}, {}
    scale = max(1.0, np.abs(full["d"]["c_lambda"]).max(), np.abs(full["d"]["lim_lambda"]).max())
    for c in checkpoints:
        r = rig.run(max_iter=c, **base)
        assert (r["same"] == full["same"]).all()
        rk[c], r64[c], r32[c] = r["resid"], r["d"]["resid"], r["d32"]["resid"]
    sides = (("kernel", full["st"], full["it"], rk), ("f64 oracle", full["d"]["status"], full["d"]["iters"], r64),
             ("f32 oracle", full["d32"]["status"], full["d32"]["iters"], r32))
    for side, st, it, res in sides:
        pst, pit = _predicted_exit(res, checkpoints, reg, max_iter, rig.n)
        bad = has & ((st != pst) | (it != pit))
        assert not bad.any(), f"{label}: {side} exits against its own checkpoint updates in envs {np.where(bad)[0][:8]}: " \
                              f"{list(zip(st[bad][:4].tolist(), it[bad][:4].tolist()))} expected {list(zip(pst[bad][:4].tolist(), pit[bad][:4].tolist()))}"
    zk = np.array([rk[c] == 0 for c in checkpoints] or np.zeros((0, rig.n), bool))
    z64 = np.array([r64[c] == 0 for c in checkpoints] or np.zeros((0, rig.n), bool))
    z32 = np.array([r32[c] == 0 for c in checkpoints] or np.zeros((0, rig.n), bool))
    differ = has & (zk != z64).any(0)
    differ32 = has & (z32 != z64).any(0)
    agree = has & ~differ
    first = 2 * w if reg == 0 else 3 * w                  # the nominal exit: the first checkpoint that can end the solve
    nominal = (STALLED, first) if first <= max_iter else (MAXITER, max_iter)
    at_nominal = has & (full["st"] == nominal[0]) & (full["it"] == nominal[1])
    print(f"     {label:34s} | envs with rows {has.sum():3d}, at {nominal} {at_nominal.sum():3d} | kernel (status, sweeps) "
          f"{sorted(set(zip(full['st'][has].tolist(), full['it'][has].tolist())))[:6]} | exact zeros at a checkpoint: kernel "
          f"{int((has & zk.any(0)).sum())}, f64 oracle {int((has & z64.any(0)).sum())}; where only one side is 0: kernel vs f64 {differ.sum()}, "
          f"f32 oracle vs f64 {differ32.sum()}")
    assert (full["st"][agree] == full["d"]["status"][agree]).all() and (full["it"][agree] == full["d"]["iters"][agree]).all(), label
    # up to the first checkpoint where only one side's update is exactly 0 the two solves took the same path; there the other side's
    # update is at rounding level: the same fixed point to float32 resolution
    k0 = np.argmax(zk != z64, axis=0) if checkpoints else np.zeros(rig.n, int)
    for e in np.where(differ)[0]:
        c = checkpoints[k0[e]]
        other = r64[c][e] if zk[k0[e], e] else rk[c][e]
        assert other <= 1e-6 * scale, f"{label}: env {e} checkpoint {c}: update {other:.2e} where the other side's is exactly 0"
    # the kernel lands exactly on such a fixed point about as often as the float32 build of the oracle does
    assert differ.sum() <= 2 * differ32.sum() + 8, label
    if nominal[0] == MAXITER:
        assert (at_nominal == has).all(), label
    _no_rows_report_nothing(full)


@pytest.mark.parametrize("name,terrain", CASE_TERRAINS)
def test_solver_exits(capi, monkeypatch, name, terrain):
    """stall_ratio = 0 and threshold = 0: every stagnation check from sweep 2w on fails unless its largest update is exactly 0, so with
    stall_reg > 0 the solve turns compliant at sweep 2w and ends STALLED at 3w, with stall_reg = 0 it ends STALLED at 2w, and a
    max_iter below that ends it MAXITER (exactly, in every environment).  A stiff compliant set (stall_reg 100) after the switch lets
    a loose threshold end some solves CONVERGED_COMPLIANT, on both sides."""
    rig = _Rig(capi, monkeypatch, name, terrain, _seed(name, terrain, 7))
    print(f"\n{name} {terrain}: {launch_config(capi, rig.bt)}")
    for w in (1, 2, 3, 8):
        _exits(rig, w, 0.02, 5 * w, f"w {w} stall_reg 0.02")
        _exits(rig, w, 0.0, 4 * w, f"w {w} stall_reg 0")
        _exits(rig, w, 0.02, 3 * w - 1, f"w {w} stall_reg 0.02 max_iter {3 * w - 1}")
        if w > 1:
            _exits(rig, w, 0.0, 2 * w - 1, f"w {w} stall_reg 0 max_iter {2 * w - 1}")
    for thr in (1e-4, 1e-5):
        r = rig.run(threshold=thr, stall_ratio=0.0, stall_window=3, stall_reg=100.0)
        s, st, s64 = r["same32"], r["st"], r["d"]["status"]
        print(f"     w 3 stall_reg 100 threshold {thr:.0e}: status gpu {np.bincount(st[s], minlength=4).tolist()} oracle "
              f"{np.bincount(s64[s], minlength=4).tolist()} f32 oracle {np.bincount(r['d32']['status'][s], minlength=4).tolist()}")
        assert (st[s] == COMPLIANT).sum() > 0 and (s64[s] == COMPLIANT).sum() > 0
        assert (st[s] == s64[s]).mean() > 0.95
        _no_rows_report_nothing(r)


# ---- 5: friction and restitution edges ----------------------------------------------------------------------------------------------

@pytest.mark.parametrize("mu", [0.0, 0.3, 2.5])
@pytest.mark.parametrize("name,terrain", CASE_TERRAINS)
def test_friction_coefficient(capi, monkeypatch, name, terrain, mu):
    """the batch's default friction in the cone of every contact (the cone checks use the mu in force); frictionless contacts carry
    no tangential impulse, on either side"""
    out = _compare(capi, monkeypatch, name, terrain, 8, dict(mu=mu))
    if mu == 0.0:
        on, d = out["on"], out["d"]
        lam = np.abs(out["ln_gpu"][on])
        assert (out["lt"][on] <= 1e-6 * lam + 1e-12).all(), f"largest tangential impulse {out['lt'][on].max():.2e}"
        assert np.abs(d["c_lambda"][:, :, :2]).max() <= 1e-12 * max(1.0, np.abs(d["c_lambda"]).max())


@pytest.mark.parametrize("name,terrain", CASE_TERRAINS)
def test_full_restitution(capi, monkeypatch, name, terrain):
    """restitution 1 from any approach speed (rest_threshold 0): every closing contact's target speed is its approach speed reversed"""
    _compare(capi, monkeypatch, name, terrain, 9, dict(restitution=1.0, rest_threshold=0.0))


# ---- 6: outputs that depend on dt -----------------------------------------------------------------------------------------------------

@pytest.mark.parametrize("name", list(CASES))
def test_contact_force_means_at_another_time_step(capi, monkeypatch, name):
    """at dt = 0.005 the per-body mean contact force of a one-sub-step launch is the scatter of its contact records times
    1 / (1 * dt), bit for bit (tests/test_gpu_contact_forces.py checks the same at the default dt)"""
    dt = 0.005
    t, bt, *_ = _batch(capi, monkeypatch, name, 256, "hm", _seed(name, "hm", 10), params=dict(dt=dt))
    bodies = list(range(t["nb"]))
    bt.set_contact_bodies(bodies)
    for k in range(3):
        bt.integrate(1)
        f, s = bt.body_contact_forces()
        ct, cnt = bt.contacts()
        fr, sr = _scatter_records(ct, cnt, bodies, dt)
        assert cnt.sum() > 64
        assert (s == sr).all()
        assert f.tobytes() == fr.tobytes(), f"sub-step {k}: largest difference {np.abs(f - fr).max():.3e}"


# ---- 7: set_params semantics --------------------------------------------------------------------------------------------------------

def _outputs(bt):
    g, v = bt.get_state(); ct, cnt = bt.contacts()
    return dict(gc=g, gv=v, contacts=ct, ncontacts=cnt, points=bt.contact_points(), iters=bt.solver_iterations(), resid=bt.solver_residual(),
                status=bt.solver_status(), tau=bt.generalized_force())


def _same_bits(x, y, label):
    for key in x:
        assert x[key].tobytes() == y[key].tobytes(), f"{label}: {key} differs"


def test_get_params_returns_what_was_set(capi, monkeypatch):
    _, bt, *_ = _batch(capi, monkeypatch, "anymal", 32, "ground", 11)
    fresh = capi.Params()
    assert capi.lib().rsb_params_default(ctypes.byref(fresh)) == 0
    p = capi.Params(0.00314159, (ctypes.c_float * 3)(0.1, -0.2, -9.7), 0.017, 1.1, 0.35, 0.97, 77, 3.3e-7, 0.61, 0.25, 0.07, 5, 0.45, 0, 2, 4, 0.013)
    assert capi.lib().rsb_batch_set_params(bt.h, ctypes.byref(p)) == 0
    back = bt.get_params()
    assert bytes(back) == bytes(p)
    # the defaults of this file are rsb_params_default with the parity tests' threshold
    for k, v in DEFAULTS.items():
        got = fresh.gravity["xyz".index(k[1])] if k in ("gx", "gy", "gz") else getattr(fresh, k)
        assert got == (np.float32(v) if isinstance(got, float) else v), k


@pytest.mark.parametrize("name", ["anymal", "atlas", "anymal_generic"])
def test_set_params_of_get_params_changes_nothing(capi, monkeypatch, name):
    """set_params(get_params()) between control steps: every output bit as in a batch that never made the call"""
    runs = []
    for touch in (False, True):
        _, bt, *_ = _batch(capi, monkeypatch, name, 256, "hm", _seed(name, "hm", 12), params=dict(dt=0.004, mu=0.7, gz=-8.0))
        outs = []
        for k in range(3):
            if touch:
                p = bt.get_params()
                assert capi.lib().rsb_batch_set_params(bt.h, ctypes.byref(p)) == 0
            bt.integrate(2)
            outs.append(_outputs(bt))
        runs.append(outs)
    for k, (x, y) in enumerate(zip(*runs)):
        _same_bits(x, y, f"control step {k}")


@pytest.mark.parametrize("name", list(CASES))
def test_params_changed_between_control_steps(capi, monkeypatch, name):
    """two control steps at the defaults, then new parameters (dt, gravity, friction, ERP, solver schedule) for two more: the change
    takes effect from the next launch, as in an oracle that makes the same change between the same calls.  The 4 worst robots are left
    out of the tail: a stagnation exit one checkpoint apart under the new stall_window sends a solve down another path."""
    t, bt, o64, o32, gc, gv, kp, kd, pt, cfg = _batch(capi, monkeypatch, name, 256, "ground", _seed(name, "ground", 13))
    kw = dict(ptarget=pt.astype(np.float64), vtarget=np.zeros((256, t["nv"])), kp=kp, kd=kd)
    a, b, c, e_ = gc.copy(), gv.copy(), gc.copy(), gv.copy()
    bt.integrate(2)
    o64.step(a, b, n_steps=2, **kw); o32.step(c, e_, n_steps=2, **kw)
    g2, _ = bt.get_state()
    e2 = np.abs(g2 - a).max(1)
    new = dict(dt=0.004, gx=1.0, gy=0.5, gz=-7.0, mu=0.5, erp=0.05, alpha_init=0.9, alpha_min=0.7, alpha_decay=0.95, stall_window=6, accel_start=4)
    bt.set_params(gravity=(new["gx"], new["gy"], new["gz"]), **{k: v for k, v in new.items() if k not in ("gx", "gy", "gz")})
    assert bt.get_state()[0].tobytes() == g2.tobytes()         # set_params launches nothing
    for o in (o64, o32):
        o.set_params(**new)
    bt.integrate(2)
    o64.step(a, b, n_steps=2, **kw); o32.step(c, e_, n_steps=2, **kw)
    gN, _ = bt.get_state()
    e = np.sort(np.abs(gN - a).max(1))[:-4]; ef = np.abs(c - a).max(1)
    print(f"{name}: after the change gc err median {np.median(e):.1e} p90 {np.quantile(e, .9):.1e} p99 {np.quantile(e, .99):.1e} "
          f"(f32 oracle p99 {np.quantile(ef, .99):.1e}); before it median {np.median(e2):.1e}")
    assert np.isfinite(gN).all()
    grow = 0.004 / 0.0025
    assert np.median(e) < 2e-5 * grow and np.median(e) < 5 * np.median(ef) + 1e-6
    assert np.quantile(e, 0.9) < max(1e-4 * grow, 5 * np.quantile(ef, 0.9))
    assert np.quantile(e, 0.99) < max(5e-3 * grow, 5 * np.quantile(ef, 0.99))


# ---- 8: refusals --------------------------------------------------------------------------------------------------------------------

FLOATS = ("dt", "erp", "alpha_init", "alpha_min", "alpha_decay", "threshold", "mu", "restitution", "rest_threshold", "stall_ratio", "stall_reg")
REFUSED = ([(f, v) for f in FLOATS for v in (float("nan"), float("inf"), float("-inf"))]
           + [("gravity", g) for g in ((float("nan"), 0.0, -9.81), (0.0, float("inf"), -9.81), (0.0, 0.0, float("-inf")))]
           + [("dt", 0.0), ("dt", -0.001), ("max_iter", 0), ("max_iter", -3), ("mu", -0.1), ("accel_m", 1), ("accel_m", 3), ("accel_m", -2),
              ("stall_reg", -0.01)]
           + [(("accel_m", "accel_start"), (2, s)) for s in (2, 0, -1)])


def test_refused_params_change_nothing(capi, monkeypatch):
    """every invalid parameter set raises RsbError, leaves get_params as it was and the next step bit-identical to a batch that never
    received the call"""
    name = "anymal"
    pair = [_batch(capi, monkeypatch, name, 64, "hm", 14, params=dict(dt=0.003, mu=0.7))[1] for _ in range(2)]
    touched, clean = pair
    for field, value in REFUSED:
        before = bytes(touched.get_params())
        kw = dict(zip(field, value)) if isinstance(field, tuple) else {field: value}
        with pytest.raises(capi.RsbError):
            touched.set_params(**kw)
        assert bytes(touched.get_params()) == before, f"{kw}: get_params changed"
        touched.integrate(1); clean.integrate(1)
        _same_bits(_outputs(touched), _outputs(clean), f"after the refused {kw}")
    # a non-finite float field is named in the message
    with pytest.raises(capi.RsbError, match="threshold is not finite"):
        touched.set_params(threshold=float("nan"))
    # and accel_start < 3 is accepted without the accelerated sweeps
    touched.set_params(accel_m=0, accel_start=1)
