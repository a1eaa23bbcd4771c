"""Every compiled instance of the step kernel against the oracle (run on an H100: pytest -m gpu).

rsb_step_kernel is a template: batch.cu dispatch_spec launches the quadruped instance (the 4 x 3-chain arithmetic compiled in) with one
or two candidate slots per lane, the humanoid instance, and the generic instance (dimensions read from the blob header) with one or two
slots, each compiled for 28, 16, 14, 8, 4 and 1 warps per CTA.  The models of tests/helpers.py reach each instance; every test asserts
through rsb_internal_launch_config that it ran the instance and the warps per CTA it names (RSB_FORCE_WPC is dropped without a
message when the CTA does not fit in shared memory).  Tolerances are those of tests/test_gpu_parity.py, scaled against the float32
build of the oracle where that test does.
"""
import os

import numpy as np
import pytest

from helpers import (ANYMAL_GC0, MAX32, MARGIN, THRESH, ROW_BIAS, OPTIONS, CASES, FITS, setup_batch, index_parity, launch_config, _batch,
                     _row, step_and_trajectory)
from oracle.oracle import Oracle
from oracle.urdf_tables import load_tables

pytestmark = pytest.mark.gpu

SUBSTEPS = 4

@pytest.fixture(scope="module")
def capi():
    import torch
    assert torch.cuda.is_available(), "GPU tests need a CUDA device"
    from raisimlib_b200 import capi as c
    return c


def _path(urdf):
    from conftest import RSC
    return os.path.join(RSC, urdf) if urdf.endswith(".urdf") else urdf


@pytest.mark.parametrize("name", list(CASES))
def test_instance_stage_outputs(capi, monkeypatch, name):
    """FK, CRBA and RNEA through integrate1() + the lazy getters against the float64 oracle, at the tolerances of
    tests/test_gpu_parity.py::test_stage_outputs_fk_crba_rnea, from random poses (any orientation, joints within +-0.5)"""
    urdf, generic, inst, base_z, q = CASES[name]
    monkeypatch.setenv("RSB_FORCE_GENERIC", "1" if generic else "0")
    monkeypatch.delenv("RSB_FORCE_WPC", raising=False)
    t, bt, o64, o32, gc, gv, tau = setup_batch(capi, urdf, 128, seed=11, base_z=base_z, tau_scale=1.0)
    cfg = launch_config(capi, bt)
    assert (cfg["spec"], cfg["slots"]) == inst, f"{name}: runs instance {cfg}, expected (spec, slots) = {inst}"
    bt.integrate1()
    M, h = bt.mass_matrix(), bt.nonlinearities()
    R, p = bt.body_poses()
    d = o64.step(gc.copy(), gv.copy(), tau_ff=tau, debug=True)
    Ms, hs = np.abs(d["M"]).max(), np.abs(d["h"]).max()
    eM, eh = np.abs(M - d["M"]).max(), np.abs(h - d["h"]).max()
    eR, ep = np.abs(R - d["R"]).max(), np.abs(p - d["p"]).max()
    print(f"{name} stage errors: M {eM:.2e}/{Ms:.1e}  h {eh:.2e}/{hs:.1e}  R {eR:.2e}  p {ep:.2e}")
    assert eR < 3e-6 and ep < 5e-6                     # float32 pose chain
    assert eM < 2e-6 * Ms                               # relative to the largest entry (total mass)
    assert eh < 2e-6 * max(hs, 1.0) * 10
    assert np.allclose(M, np.transpose(M, (0, 2, 1)))


# every case on both terrains, and the row bias of stage C (ERP, restitution) on the humanoid and a generic instance
STEP_CASES = [pytest.param(name, terrain, None, id=f"{name}-{terrain}") for name in CASES for terrain in ("ground", "hm")] + [
    pytest.param("atlas", "ground", ROW_BIAS, id="atlas-ground-bias"), pytest.param("anymal_generic", "hm", ROW_BIAS, id="anymal_generic-hm-bias")]


@pytest.mark.parametrize("name,terrain,bias", STEP_CASES)
def test_instance_step_and_trajectory(capi, monkeypatch, name, terrain, bias):
    """one step (contact lists, state, impulses, complementarity) and 10 steps (state) against the oracle, PD targets on, joints at
    their stops and actuators at their effort limits"""
    step_and_trajectory(capi, monkeypatch, name, terrain, seed=1000 + 17 * len(name) + (terrain == "hm"), params=bias)


def _sweep_n(sms):
    """a batch size at which every warps-per-CTA option runs at least two rounds and ends on a partly filled CTA"""
    n = int(1.35 * 28 * sms)
    while True:
        ok = True
        for w in OPTIONS:
            T = w * (2 * sms if w == 14 else sms)
            rounds = -(-n // T)
            ok &= rounds >= 2 and (w == 1 or (n - (rounds - 1) * T) % w != 0)
        if ok:
            return n
        n += 1


def _run_outputs(capi, bt, t, n, targets):
    obs = np.empty((n, bt.ob_dim()), np.float32)
    out = []
    for tg in targets:
        bt.control_step(tg.copy(), SUBSTEPS, obs)
        g, v = bt.get_state(); rec, cnt = bt.contacts()
        out.append(dict(obs=obs.copy(), gc=g, gv=v, contacts=rec, ncontacts=cnt, points=bt.contact_points(), iters=bt.solver_iterations(),
                        resid=bt.solver_residual(), status=bt.solver_status(), tau=bt.generalized_force()))
    return out


@pytest.mark.parametrize("name", list(CASES))
def test_warps_per_cta_bit_identical(capi, monkeypatch, name):
    """One warp per environment: the CTA size decides where and when an environment is computed, never what.  Every option that fits
    gives the default pick's outputs bit for bit after 4 control steps of 4 sub-steps on the rough map; the default pick is compared
    with the oracle on a sample that holds the first and last environment of every round."""
    monkeypatch.setenv("RSB_FORCE_WPC", "1")
    probe = capi.Batch(capi.Model(_path(CASES[name][0])), 100000)
    sms = launch_config(capi, probe)["grid"]           # one-warp CTAs: one per SM
    del probe
    n = _sweep_n(sms)
    runs, taken = {}, []
    for w in (None,) + OPTIONS:
        t, bt, o64, o32, gc, gv, kp, kd, pt, cfg = _batch(capi, monkeypatch, name, n, "hm", seed=2000 + len(name), wpc=w)
        rng = np.random.default_rng(7)
        targets = [pt + np.float32(0.1) * rng.uniform(-1, 1, pt.shape).astype(np.float32) for _ in range(4)]
        if w is not None:
            if cfg["wpc"] != w:                      # did not fit: pick_config kept its own choice
                continue
            taken.append(w)
        T = cfg["wpc"] * cfg["grid"]
        rounds = -(-n // T)
        assert rounds >= 2 and (cfg["wpc"] == 1 or (n - (rounds - 1) * T) % cfg["wpc"] != 0)
        runs[w] = (cfg, _run_outputs(capi, bt, t, n, targets))
        if w is None:
            ref_cfg = cfg
            first = np.arange(rounds) * T
            last = np.minimum(first + T, n) - 1
            idx = np.unique(np.r_[first, last, np.random.default_rng(3).choice(n, 256 - 2 * rounds, replace=False)])
            a, b = gc[idx].copy(), gv[idx].copy(); c, e_ = gc[idx].copy(), gv[idx].copy()
            vt = np.zeros((len(idx), t["nv"]))
            crmax = 0
            for tg in targets:
                for s in range(SUBSTEPS):
                    d = o64.step(a, b, ptarget=tg[idx].astype(np.float64), vtarget=vt, kp=kp, kd=kd, debug=True)
                    crmax = max(crmax, int((3 * d["ncontacts"] + d["nlimits"]).max()))
                o32.step(c, e_, n_steps=SUBSTEPS, ptarget=tg[idx].astype(np.float64), vtarget=vt, kp=kp, kd=kd)
            out = runs[None][1][-1]
            e = np.abs(out["gc"][idx] - a).max(1); ef = np.abs(c - a).max(1)
            _row(name, cfg, n, out["ncontacts"].mean(), crmax, f"default pick, {len(idx)} sampled envs vs oracle after 16 sub-steps: gc err "
                 f"median {np.median(e):.1e} p90 {np.quantile(e, .9):.1e} p99 {np.quantile(e, .99):.1e} (f32 oracle p99 {np.quantile(ef, .99):.1e})")
            assert np.isfinite(out["gc"]).all() and out["ncontacts"].mean() > 0.5
            # 16 sub-steps of robots landing on rough ground under stiff PD: contact-set changes one sub-step apart are bounded by
            # the float32 build of the oracle itself, as in test_trajectory_50_steps
            assert np.median(e) < 2e-5 and np.median(e) < 5 * np.median(ef) + 1e-6
            assert np.quantile(e, 0.9) < max(1e-4, 5 * np.quantile(ef, 0.9))
            assert np.quantile(e, 0.99) < max(5e-3, 5 * np.quantile(ef, 0.99))
        else:
            _row(name, cfg, n, runs[w][1][-1]["ncontacts"].mean(), -1, f"forced WPC {w}, compared bit for bit with the default pick")
        del bt
    assert tuple(taken) == FITS[name], f"{name}: warps per CTA that fit {taken}, expected {FITS[name]}"
    assert ref_cfg["wpc"] in taken
    for w in taken:
        for k, (x, y) in enumerate(zip(runs[None][1], runs[w][1])):
            for key in x:
                assert x[key].shape == y[key].shape and x[key].tobytes() == y[key].tobytes(), \
                    f"{name}: control step {k}: {key} differs between {runs[w][0]['wpc']} warps per CTA and the default {ref_cfg['wpc']}"


def _kept_is_deepest(pts, cnt, dgpu, d):
    """each list holds the reference's 8 deepest candidates; the only allowed difference is a swap of candidates whose depths tie
    with the cut-off (the shallowest kept one) to MARGIN"""
    bad = 0
    for e in range(len(cnt)):
        if (pts[e] == d["c_pt"][e]).all():
            continue
        g = {int(k): float(x) for k, x in zip(pts[e], dgpu[e]) if k >= 0}
        r = {int(k): float(x) for k, x in zip(d["c_pt"][e], d["c_depth"][e]) if k >= 0}
        cut = min(min(g.values()), min(r.values()))
        if any(abs((g[k] if k in g else r[k]) - cut) > MARGIN for k in set(g) ^ set(r)):
            bad += 1
    return bad


def test_more_than_32_penetrating_candidates(capi, monkeypatch):
    """MAX32 lying flat, sunk into the rough map: more than 32 of its 64 candidates penetrate (the second pass of stage B's ranking
    loop, a hit list past row 32), and 4 of its in-plane joints are past their stops, so the solve has 3 x 8 + 4 = 28 rows"""
    monkeypatch.delenv("RSB_FORCE_GENERIC", raising=False); monkeypatch.delenv("RSB_FORCE_WPC", raising=False)
    n = 64
    t = load_tables(MAX32)
    bt = capi.Batch(capi.Model(MAX32), n)
    cfg = launch_config(capi, bt)
    assert (cfg["spec"], cfg["slots"]) == (0, 2)
    rng = np.random.default_rng(4242)
    xs, ys = 65, 49
    H = (0.03 * rng.uniform(-1, 1, (ys, xs))).astype(np.float32)
    bt.set_heightmap(xs, ys, 12.8, 9.6, 0.1, -0.2, H)
    prm = dict(threshold=THRESH)
    bt.set_params(**prm)
    o64, o32 = Oracle(t, params=prm), Oracle(t, precision="f32", params=prm)
    for o in (o64, o32):
        o.set_heightmap(xs, ys, 12.8, 9.6, 0.1, -0.2, H.astype(np.float64))
    gc = np.zeros((n, t["nq"])); gc[:, :2] = rng.uniform(-3, 3, (n, 2)); gc[:, 2] = -0.03
    yaw = rng.uniform(-np.pi, np.pi, n); gc[:, 3] = np.cos(yaw / 2); gc[:, 6] = np.sin(yaw / 2)
    gc[:, 7:] = rng.uniform(-0.02, 0.02, (n, t["nq"] - 7))
    roots = [t["qidx"][t["body_names"].index(f"c{c}_l1")] for c in range(5)]      # turn about the base normal: the star stays flat
    gc[:, roots[:4]] = rng.choice([-0.6, 0.6], (n, 4))                             # beyond (-0.5, 0.5)
    gc32 = gc.astype(np.float32)
    bt.set_state(gc32, np.zeros((n, t["nv"]), np.float32))
    bt.integrate(1)
    g1, v1 = bt.get_state(); ct, cnt = bt.contacts(); pts = bt.contact_points(); st = bt.solver_status()
    a, b = gc32.astype(np.float64), np.zeros((n, t["nv"]))
    d32 = o32.step(a.copy(), b.copy(), debug=True)
    d = o64.step(a, b, debug=True)
    # penetrating for certain: point candidates whose lowest point is below the lowest height of the map (oracle poses)
    P = d["p"][:, t["pt_body"]] + np.einsum("ebij,bj->ebi", d["R"][:, t["pt_body"]], t["pt_pos"])
    deep = ((P[:, :, 2] - t["pt_rad"][None, :] < H.min()) & (t["pt_type"] == 0)[None, :]).sum(1)
    print(f"MAX32 sunk in the rough map: penetrating candidates >= {deep.min()} (mean {deep.mean():.1f}); K {cnt.mean():.2f}; oracle limit rows "
          f"{np.bincount(d['nlimits'], minlength=5).tolist()}; kept candidates >= 32: {int((pts >= 32).sum())}")
    assert (deep > 32).all()
    assert (cnt == 8).all() and (d["nlimits"] == 4).all()
    assert _kept_is_deepest(pts, cnt, ct["depth"], d32) == 0
    assert (np.diff(np.where(pts >= 0, pts, 10**6), axis=1) > 0).all()          # candidate order
    same = (pts == d["c_pt"]).all(1)
    conv = same & (st == 0) & (d["status"] == 0)
    ev = np.abs(v1 - b)[conv].max(1)
    print(f"   one step, CR = 28: solver status gpu {np.bincount(st, minlength=4).tolist()} oracle {np.bincount(d['status'], minlength=4).tolist()} "
          f"(converged / on the compliant set / stalled / max_iter); gv err median {np.median(ev):.1e} max {ev.max():.1e} on {conv.sum()} envs converged on both sides")
    # a 32-body star pressed 10 cm into rough ground with four stops engaged: the exact contact set often ends on the compliant set
    assert conv.mean() > 0.5 and ((st == 1) == (d["status"] == 1)).mean() > 0.9
    assert np.median(ev) < 5e-5 and np.quantile(ev, 0.99) < 5e-3


def test_quadruped_largest_constraint_problem(capi, monkeypatch):
    """the ANYmal-like robot lying on its belly with all four HAA joints past their stops: 8 contacts and 4 joint-limit rows, the
    largest Gauss-Seidel problem (CR = 28), in the quadruped instance; one step against the oracle"""
    monkeypatch.delenv("RSB_FORCE_GENERIC", raising=False); monkeypatch.delenv("RSB_FORCE_WPC", raising=False)
    n = 128
    path = _path("anymal_c_like.urdf")
    t = load_tables(path)
    bt = capi.Batch(capi.Model(path), n)
    cfg = launch_config(capi, bt)
    assert (cfg["spec"], cfg["slots"]) == (1, 2)
    prm = dict(threshold=THRESH)
    bt.set_ground(0.0); bt.set_params(**prm)
    o64, o32 = Oracle(t, params=prm), Oracle(t, precision="f32", params=prm)
    for o in (o64, o32):
        o.set_ground(0.0)
    rng = np.random.default_rng(99)
    gc = np.tile(ANYMAL_GC0, (n, 1)); gc[:, :2] = rng.uniform(-2, 2, (n, 2)); gc[:, 2] = rng.uniform(0.05, 0.07, n)
    yaw = rng.uniform(-np.pi, np.pi, n); gc[:, 3] = np.cos(yaw / 2); gc[:, 6] = np.sin(yaw / 2)
    haa = [7, 10, 13, 16]
    gc[:, haa] = np.where(rng.uniform(size=(n, 4)) < 0.5, rng.uniform(0.55, 0.7, (n, 4)), rng.uniform(-0.9, -0.78, (n, 4)))   # beyond (-0.72, 0.49)
    gc[:, [8, 11, 14, 17]] = rng.choice([-1.5, 1.5], (n, 4))           # thighs out flat
    gc[:, [9, 12, 15, 18]] = rng.uniform(-0.3, 0.3, (n, 4))
    gc32 = gc.astype(np.float32)
    bt.set_state(gc32, (0.1 * rng.standard_normal((n, 18))).astype(np.float32))
    gv = bt.get_state()[1].astype(np.float64)
    bt.integrate(1)
    g1, v1 = bt.get_state(); ct, cnt = bt.contacts(); pts = bt.contact_points(); st = bt.solver_status()
    a, b = gc32.astype(np.float64), gv.copy()
    d32 = o32.step(a.copy(), b.copy(), debug=True)
    d = o64.step(a, b, debug=True)
    full = (cnt == 8) & (d["nlimits"] == 4)
    print(f"ANYmal-like on its belly: K hist {np.bincount(cnt, minlength=9).tolist()}, oracle limit rows {np.bincount(d['nlimits'], minlength=5).tolist()}, "
          f"CR = 28 in {full.sum()} of {n} envs")
    assert full.mean() > 0.5
    hard = index_parity(pts, cnt, d32, "anymal on its belly")
    assert not hard.any()
    conv = (pts == d["c_pt"]).all(1) & (st == 0) & (d["status"] == 0)
    assert (conv & full).mean() > 0.4
    ev = np.abs(v1 - b)[conv & full].max(1)
    print(f"   one step, CR = 28: gv err median {np.median(ev):.1e} max {ev.max():.1e}")
    assert np.median(ev) < 5e-5 and np.quantile(ev, 0.99) < 5e-3
