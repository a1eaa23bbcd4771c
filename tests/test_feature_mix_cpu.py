"""The per-environment feature composition of tests/feature_mix_ref.py against the oracle it is built on (no GPU): with every feature
off it is Oracle.step itself, and with one feature on it is what that feature's own tests compare the batch with -- the oracle of
tables_with, the oracle fed the restated delayed commands, the oracle driven by the restated network torque -- bit for bit."""
import os

import numpy as np

from actuation_delay_ref import applied
from actuator_network_ref import random_layers, shift, torque
from body_inertia_ref import randomized, rows_of, tables_with
from conftest import RSC
from feature_mix_ref import MixRef, dof_q
from helpers import ANYMAL_GC0, THRESH, effort_limits
from oracle.oracle import Oracle
from oracle.urdf_tables import load_tables

N, SUB, PRM = 6, 4, dict(threshold=THRESH)


def _anymal(seed):
    t = load_tables(os.path.join(RSC, "anymal_c_like.urdf"))
    rng = np.random.default_rng(seed)
    gc = np.tile(ANYMAL_GC0, (N, 1)); gc[:, 2] = 0.56
    gc[:, 7:] += rng.uniform(-0.15, 0.15, (N, 12))
    gv = 0.3 * rng.standard_normal((N, 18))
    kp = np.r_[np.zeros(6), 300.0 * np.ones(12)]; kd = np.r_[np.zeros(6), 4.0 * np.ones(12)]
    return t, gc, gv, kp, kd, rng


def _commands(t, rng, steps):
    """per control step: (ptarget [N, nq], vtarget [N, nv], tau_ff [N, nv]), the base parts constant"""
    out = []
    for _ in range(steps):
        pt = np.tile(ANYMAL_GC0, (N, 1)); pt[:, 7:] += rng.uniform(-0.5, 0.5, (N, 12))
        vt = np.zeros((N, 18)); vt[:, 6:] = rng.uniform(-1, 1, (N, 12))
        tau = np.zeros((N, 18)); tau[:, 6:] = rng.uniform(-8, 8, (N, 12))
        out.append((pt, vt, tau))
    return out


def _run_mix(ref, gc, gv, cmds):
    a, b = gc.copy(), gv.copy()
    for pt, vt, tau in cmds:
        for _ in range(SUB):
            ref.substep(a, b, pt, vt, tau)
    return a, b


def test_all_features_off_is_the_oracle_step():
    t, gc, gv, kp, kd, rng = _anymal(1)
    (pt, vt, tau), = _commands(t, rng, 1)
    a, b = _run_mix(MixRef(t, N, params=PRM, kp=kp, kd=kd), gc, gv, [(pt, vt, tau)])
    o = Oracle(t, params=PRM)
    o.set_ground(0.0)
    c, d = gc.copy(), gv.copy()
    o.step(c, d, n_steps=SUB, tau_ff=tau, ptarget=pt, vtarget=vt, kp=kp, kd=kd)
    assert a.tobytes() == c.tobytes() and b.tobytes() == d.tobytes()


def test_rows_alone_are_the_oracle_with_the_environment_gains_and_limits():
    t, gc, gv, kp, kd, rng = _anymal(2)
    (pt, vt, tau), = _commands(t, rng, 1)
    rows = np.full((N, 18, 3), -1.0)
    rows[:, 6:] = rng.uniform(20.0, 400.0, (N, 12, 3))
    rows[0, 7, 2] = np.inf; rows[1, 8, 0] = 0.0
    a, b = _run_mix(MixRef(t, N, params=PRM, kp=kp, kd=kd, rows=rows), gc, gv, [(pt, vt, tau)])
    lim = np.where(rows[:, :, 2] >= 0, rows[:, :, 2], effort_limits(t))
    for e in range(N):
        jeff = t["jeffort"].copy()
        for bd in range(1, t["nb"]):
            jeff[bd] = lim[e, t["vidx"][bd]]
        o = Oracle(dict(t, jeffort=jeff), params=PRM)
        o.set_ground(0.0)
        c, d = gc[e:e + 1].copy(), gv[e:e + 1].copy()
        kpe = np.where(rows[e, :, 0] >= 0, rows[e, :, 0], kp); kpe[:6] = 0
        kde = np.where(rows[e, :, 1] >= 0, rows[e, :, 1], kd); kde[:6] = 0
        o.step(c, d, n_steps=SUB, tau_ff=tau[e:e + 1], ptarget=pt[e:e + 1], vtarget=vt[e:e + 1], kp=kpe, kd=kde)
        assert a[e].tobytes() == c[0].tobytes() and b[e].tobytes() == d[0].tobytes(), f"environment {e}"


def test_inertia_alone_is_the_tables_with_oracle():
    t, gc, gv, kp, kd, rng = _anymal(3)
    (pt, vt, tau), = _commands(t, rng, 1)
    sets = [randomized(t, rng) for _ in range(N)]
    rows = np.stack([rows_of(*s) for s in sets]).astype(np.float64)
    a, b = _run_mix(MixRef(t, N, params=PRM, kp=kp, kd=kd, inertia=rows), gc, gv, [(pt, vt, tau)])
    for e in range(N):
        o = Oracle(tables_with(t, *sets[e]), params=PRM)
        o.set_ground(0.0)
        c, d = gc[e:e + 1].copy(), gv[e:e + 1].copy()
        o.step(c, d, n_steps=SUB, tau_ff=tau[e:e + 1], ptarget=pt[e:e + 1], vtarget=vt[e:e + 1], kp=kp, kd=kd)
        assert a[e].tobytes() == c[0].tobytes() and b[e].tobytes() == d[0].tobytes(), f"environment {e}"


def test_delay_alone_is_the_oracle_fed_the_restated_commands():
    """delays 0 .. 16 over 40 sub-steps, and one environment's history emptied at sub-step 20 with a new delay"""
    t, gc, gv, kp, kd, rng = _anymal(4)
    steps = 10
    cmds = _commands(t, rng, steps)
    delay = np.array([0, 1, 3, 7, 16, 5])
    ref = MixRef(t, N, params=PRM, kp=kp, kd=kd, delay=delay)
    a, b = gc.copy(), gv.copy()
    for k, (pt, vt, tau) in enumerate(cmds):
        if k == 5:
            ref.empty_delay_history([2]); ref.delay[2] = 11
        for _ in range(SUB):
            ref.substep(a, b, pt, vt, tau)
    o = Oracle(t, params=PRM)
    o.set_ground(0.0)
    per_sub = [np.repeat(np.stack([c[i] for c in cmds]), SUB, axis=0) for i in range(3)]      # [T, N, w]
    app = [np.empty_like(p) for p in per_sub]
    d_of = np.tile(delay[None, :], (steps * SUB, 1)); d_of[5 * SUB:, 2] = 11
    for e in range(N):
        for i in range(3):
            app[i][:, e] = applied(per_sub[i][:, e], d_of[:, e], {5 * SUB} if e == 2 else ())
    c, d = gc.copy(), gv.copy()
    for s in range(steps * SUB):
        o.step(c, d, tau_ff=app[2][s], ptarget=app[0][s], vtarget=app[1][s], kp=kp, kd=kd)
    assert a.tobytes() == c.tobytes() and b.tobytes() == d.tobytes()
    # the delays were seen: the undelayed composition ends elsewhere
    e_, f_ = _run_mix(MixRef(t, N, params=PRM, kp=kp, kd=kd), gc, gv, cmds)
    assert (e_[delay > 0] != a[delay > 0]).any(1).all()


def test_network_alone_is_the_oracle_driven_by_the_restated_torque():
    """a network on four non-adjacent joint dofs, its history zero at the start, 8 sub-steps"""
    t, gc, gv, kp, kd, rng = _anymal(5)
    cmds = _commands(t, rng, 2)
    dofs = np.array([6, 9, 10, 17])
    layers = random_layers(np.random.default_rng(6), 3, 2, 32)
    ref = MixRef(t, N, params=PRM, kp=kp, kd=kd, network=(dofs, layers, 3))
    a, b = gc.copy(), gv.copy()
    nets = []
    for pt, vt, tau in cmds:
        for _ in range(SUB):
            nets.append(ref.substep(a, b, pt, vt, tau)["tau_net"])
    o = Oracle(t, params=PRM)
    o.set_ground(0.0)
    kpn, kdn = kp.copy(), kd.copy(); kpn[dofs] = 0.0; kdn[dofs] = 0.0
    q = dof_q(t)[dofs]
    lim = effort_limits(t)[dofs]
    c, d = gc.copy(), gv.copy()
    hist = np.zeros((N, len(dofs), 2, 2))
    for k, (pt, vt, tau) in enumerate(cmds):
        for s in range(SUB):
            e, v = pt[:, q] - c[:, q], d[:, dofs]
            tf = tau.copy(); tf[:, dofs] = torque(layers, e, v, hist, tau[:, dofs], lim)
            assert tf[:, dofs].tobytes() == nets[k * SUB + s].tobytes()
            hist = shift(e, v, hist)
            o.step(c, d, tau_ff=tf, ptarget=pt, vtarget=vt, kp=kpn, kd=kdn)
    assert a.tobytes() == c.tobytes() and b.tobytes() == d.tobytes()
    assert ref.hist.tobytes() == hist.tobytes()
    assert np.abs(np.concatenate(nets)).max() > 5.0
