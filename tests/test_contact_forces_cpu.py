"""The reference of the per-body contact forces (tests/contact_force_ref.py) pinned on the CPU, float64 oracle, before it judges the
kernel (tests/test_gpu_contact_forces.py): known answers, impulse-momentum balance, action = reaction of self contacts."""
import numpy as np
import pytest

from contact_force_ref import scatter_step, step_with_forces, tangent_frame
from helpers import SPHERE_URDF
from oracle.oracle import Oracle
from oracle.self_oracle import SelfOracle
from oracle.urdf_tables import load_tables
from test_self_collision_oracle import anymal_leg_pairs, crossed_anymal

G, DT = 9.81, 0.0025


def _drop(t, n, rng, z):
    gc = np.zeros((n, t["nq"])); gc[:, 2] = z
    gc[:, :2] = rng.uniform(-2, 2, (n, 2))
    q = np.c_[np.ones(n), 0.3 * rng.standard_normal((n, 3))]
    gc[:, 3:7] = q / np.linalg.norm(q, axis=1, keepdims=True)
    gc[:, 7:] = rng.uniform(-0.5, 0.5, (n, t["nq"] - 7))
    return gc, 0.5 * rng.standard_normal((n, t["nv"]))


def test_tangent_frame_is_right_handed_and_switches_axis():
    n = np.array([[0, 0, 1.0], [0.95, 0, np.sqrt(1 - 0.95 ** 2)], [0.6, 0.0, 0.8]])
    t1, t2 = tangent_frame(n)
    assert np.allclose(t1[0], [1, 0, 0]) and np.allclose(t2[0], [0, 1, 0])
    assert np.allclose(t1[1], [0, 1, 0])                       # |n_x| >= 0.9: built from e_y
    for a, b in ((t1, n), (t2, n), (t1, t2)):
        assert np.abs((a * b).sum(1)).max() < 1e-15
    assert np.allclose(np.cross(t1, t2), n)


def test_substeps_one_at_a_time_equal_one_call_bit_for_bit(anymal_tables):
    """the reference steps the oracle sub-step by sub-step: that is the same trajectory as one call of n_steps (no warm start)"""
    t = anymal_tables
    rng = np.random.default_rng(5)
    gc, gv = _drop(t, 32, rng, 0.45)
    o = Oracle(t); o.set_ground(0.0)
    a, b = gc.copy(), gv.copy()
    o.step(a, b, n_steps=4)
    c, e = gc.copy(), gv.copy()
    for _ in range(4):
        o.step(c, e, n_steps=1)
    assert a.tobytes() == c.tobytes() and b.tobytes() == e.tobytes()


def test_sphere_resting_on_the_plane_carries_its_weight():
    t = load_tables(SPHERE_URDF)
    o = Oracle(t); o.set_ground(0.0)
    gc = np.array([[0, 0, 0.0999, 1, 0, 0, 0.0]]); gv = np.zeros((1, 6))
    f, steps, _ = step_with_forces(o, gc, gv, 4, [0])
    assert steps[0, 0] == 4
    assert np.abs(f[0, 0] - [0, 0, 2.0 * G]).max() < 1e-9 * 2.0 * G


def test_bounce_inside_the_control_step_shows_in_the_force_and_not_in_the_last_contact_list():
    """the sphere arrives at 1 m/s, penetrates in the first of 4 sub-steps only and leaves with restitution 0.5"""
    t = load_tables(SPHERE_URDF)
    o = Oracle(t, params=dict(restitution=0.5)); o.set_ground(0.0)
    m, vn = 2.0, -1.0
    gc = np.array([[0, 0, 0.0999, 1, 0, 0, 0.0]]); gv = np.zeros((1, 6)); gv[0, 2] = vn
    f, steps, dbg = step_with_forces(o, gc, gv, 4, [0])
    assert steps[0, 0] == 1 and [int(d["ncontacts"][0]) for d in dbg] == [1, 0, 0, 0]
    want = m * (-0.5 * vn - vn) + m * G * DT
    assert abs(f[0, 0, 2] * 4 * DT - want) < 1e-9 * want and np.abs(f[0, 0, :2]).max() < 1e-12
    assert dbg[-1]["ncontacts"][0] == 0           # what a caller reads after the launch: no contact


@pytest.mark.parametrize("which", ["anymal", "atlas"])
def test_contact_forces_balance_the_change_of_linear_momentum(which, anymal_tables, atlas_tables):
    """every body listed, random drops onto a rough map.  In each sub-step the rows 0-2 of the oracle's velocity update,
    M (v+ - v) = -dt h + J^T lambda, hold the impulses as they are (the translational rows of a contact's J^T are the identity), so
    the sum over bodies of the scattered impulses equals M[0:3] (v+ - v) + dt h[0:3] to rounding.  Over the launch,
    sum of force * substeps * dt = m (v_com+ - v_com) - m g substeps dt with m v_com = M[0:3, :] gv only to first order in dt: each
    sub-step uses M and h of the pose it starts from.  This float64 run shows 3.8e-3 of the impulse scale at worst on the quadruped
    and 5.7e-2 on the humanoid (whose feet land with seven contacts per sub-step); the bounds leave a factor 2."""
    t = anymal_tables if which == "anymal" else atlas_tables
    n, sub = 64, 4
    rng = np.random.default_rng(21)
    gc, gv = _drop(t, n, rng, 0.45 if which == "anymal" else 0.55)
    o = Oracle(t)
    H = 0.1 * rng.uniform(-1, 1, (49, 65))
    o.set_heightmap(65, 49, 12.8, 9.6, 0.1, -0.2, H)
    bodies = list(range(t["nb"]))
    mass = t["mass"].sum()
    acc, steps, exact = np.zeros((n, 3)), np.zeros((n, t["nb"]), np.int32), 0.0
    for k in range(sub):
        v0 = gv.copy()
        d = o.step(gc, gv, debug=True)
        if k == 0:
            p0 = np.einsum("eij,ej->ei", d["M"][:, 0:3, :], v0)
        imp, hit = scatter_step(d, bodies)
        row = np.einsum("eij,ej->ei", d["M"][:, 0:3, :], gv - v0) + DT * d["h"][:, 0:3]
        exact = max(exact, np.abs(imp.sum(1) - row).max() / (mass * G * DT))
        acc += imp.sum(1); steps += hit
    M1 = o.step(gc.copy(), gv.copy(), debug=True)["M"]
    p1 = np.einsum("eij,ej->ei", M1[:, 0:3, :], gv)
    rhs = p1 - p0 - mass * np.array([0, 0, -G]) * sub * DT
    err = np.abs(acc - rhs).max(1) / (np.abs(acc).max(1) + mass * G * sub * DT)
    print(f"{which}: bodies touched {int((steps > 0).any(0).sum())}, per-sub-step balance {exact:.1e}, momentum over the launch worst {err.max():.2e} median {np.median(err):.2e}")
    assert (steps > 0).any(0).sum() >= 3 and steps.max() == sub
    assert exact < 1e-9
    assert err.max() < {"anymal": 8e-3, "atlas": 0.12}[which]


def test_self_contacts_act_with_opposite_forces_on_their_two_bodies(anymal_tables):
    """legs crossed and driven into each other, no terrain, no gravity: with every body listed the forces sum to zero, and an
    environment with a single self contact shows it on exactly its two bodies, with opposite signs"""
    t = anymal_tables
    rng = np.random.default_rng(3)
    n = 16
    gc = crossed_anymal(n, rng); gv = 0.3 * rng.standard_normal((n, t["nv"]))
    o = SelfOracle(t, params=dict(gz=0.0))
    o.set_self_collision(anymal_leg_pairs())
    bodies = list(range(t["nb"]))
    kp = np.r_[np.zeros(6), 100.0 * np.ones(12)]; kd = np.r_[np.zeros(6), 2.0 * np.ones(12)]
    pt = gc.copy(); pt[:, [7, 13]] -= 0.5; pt[:, [10, 16]] += 0.5         # drive the crossed legs into each other
    d = o.step(gc, gv, ptarget=pt, vtarget=np.zeros((n, t["nv"])), kp=kp, kd=kd, debug=True)
    imp, hit = scatter_step(d, bodies)
    assert d["ncontacts"].sum() > n // 2 and (d["c_pair"][d["c_pt"] >= 0] < 0).all() and np.abs(imp).max() > 1e-3
    assert np.abs(imp.sum(1)).max() < 1e-12 * max(1.0, np.abs(imp).max())
    single = np.where(d["ncontacts"] == 1)[0]
    assert len(single) > 0
    for e in single:
        a, b = int(d["c_body"][e, 0]), -1 - int(d["c_pair"][e, 0])
        assert sorted(np.where(hit[e])[0]) == sorted((a, b))
        assert np.abs(imp[e, a] + imp[e, b]).max() < 1e-12 * max(1.0, np.abs(imp[e, a]).max())


def test_free_flight_gives_zero_force_and_no_steps(anymal_tables):
    t = anymal_tables
    rng = np.random.default_rng(8)
    gc, gv = _drop(t, 8, rng, 5.0)
    o = Oracle(t); o.set_ground(0.0)
    f, steps, _ = step_with_forces(o, gc, gv, 4, list(range(t["nb"])))
    assert not f.any() and not steps.any()
