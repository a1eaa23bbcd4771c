"""Analytic known-answer tests that pin the CPU oracle (SURVEY.md section 4(1), 4(3)).

The reference snapshot has no tests, golden vectors or fixtures for this path
(`/root/reference/.travis.yml:9-12` only builds; SURVEY 8c: parity unpinned), so the oracle
is validated against closed-form physics and an independent numpy restatement instead.
"""
import numpy as np
import pytest

from oracle.oracle import Oracle
from oracle.urdf_tables import load_tables
from helpers import (ANYMAL_GC0, PENDULUM_URDF, SPHERE_URDF, BOX_URDF, mass_matrix_numpy, potential_energy,
                     integrate_gc, random_state, fk_numpy, body_jacobians, QUAD_FEET, QUAD_PRISMATIC, QUAD_BRANCHED, HEXAPOD, MAX32)

G = 9.81
# the models that reach every compiled instance of the step kernel (tests/test_gpu_instances.py): the oracle those tests compare with
# is pinned on their shapes here first
INSTANCE_MODELS = {"quad_feet": QUAD_FEET, "quad_prismatic": QUAD_PRISMATIC, "quad_branched": QUAD_BRANCHED, "hexapod": HEXAPOD, "max32": MAX32}


def _tables(which, anymal_tables, atlas_tables):
    if which in INSTANCE_MODELS:
        return load_tables(INSTANCE_MODELS[which])
    return {"anymal": anymal_tables, "atlas": atlas_tables}.get(which) or load_tables(PENDULUM_URDF)


def test_tables_shapes(anymal_tables, atlas_tables):
    a, h = anymal_tables, atlas_tables
    assert (a["nb"], a["nq"], a["nv"]) == (13, 19, 18)
    assert (h["nb"], h["nq"], h["nv"]) == (31, 37, 36)
    assert abs(a["mass"].sum() - 50.4) < 1e-9          # fixed-joint merge keeps the total mass
    assert h["depth"].max() == 10
    # shank body absorbed the foot link through the fixed joint: its COM moved toward the foot
    i = a["body_names"].index("LF_SHANK")
    assert abs(a["mass"][i] - 0.85) < 1e-12
    m0, c0, m1, c1 = 0.6, np.array([0.03, 0.01, -0.10]), 0.25, np.array([0.088, 0.013, -0.338])
    assert np.allclose(a["com"][i], (m0 * c0 + m1 * c1) / 0.85)


def test_free_fall_closed_form(anymal_tables):
    o = Oracle(anymal_tables)
    gc = ANYMAL_GC0[None].copy(); gc[0, 2] = 10.0
    gv = np.zeros((1, 18))
    n, dt = 200, 0.0025
    o.step(gc, gv, n_steps=n)
    # semi-implicit Euler: v_k = -g k dt ; z_n = z0 - g dt^2 n(n+1)/2 ; joints do not move in free fall
    assert abs(gv[0, 2] + G * n * dt) < 1e-9
    assert abs(gc[0, 2] - (10.0 - G * dt * dt * n * (n + 1) / 2)) < 1e-9
    assert np.allclose(gc[0, 7:], ANYMAL_GC0[7:], atol=1e-9)
    assert np.allclose(gc[0, 3:7], [1, 0, 0, 0], atol=1e-12)


@pytest.mark.parametrize("which", ["anymal", "atlas", "pendulum", *INSTANCE_MODELS])
def test_mass_matrix_vs_jacobian_sum(which, anymal_tables, atlas_tables):
    t = _tables(which, anymal_tables, atlas_tables)
    o = Oracle(t)
    rng = np.random.default_rng(1)
    gc, gv = random_state(t, rng, 4, pos_scale=20.0)
    gc0 = gc.copy()
    d = o.step(gc, gv, n_steps=1, debug=True)
    for e in range(4):
        Mref = mass_matrix_numpy(t, gc0[e])
        assert np.allclose(d["M"][e], Mref, rtol=1e-10, atol=1e-10)
        assert np.allclose(d["M"][e], d["M"][e].T)
        assert np.linalg.eigvalsh(d["M"][e]).min() > 0


def test_single_pendulum_closed_form():
    urdf = """<robot name="p"><link name="world"/>
      <link name="l"><inertial><origin xyz="0 0 -0.5"/><mass value="2.0"/><inertia ixx="0.1" ixy="0" ixz="0" iyy="0.1" iyz="0" izz="0.01"/></inertial></link>
      <joint name="j" type="revolute"><parent link="world"/><child link="l"/><origin xyz="0 0 1"/><axis xyz="0 1 0"/></joint></robot>"""
    t = load_tables(urdf)
    o = Oracle(t)
    q = 0.7
    gc, gv = np.array([[q]]), np.array([[1.3]])
    d = o.step(gc, gv, n_steps=1, debug=True)
    m, l, I = 2.0, 0.5, 0.1
    assert abs(d["M"][0, 0, 0] - (I + m * l * l)) < 1e-12
    # rotation about +y by q moves the COM (0,0,-l) to (-l sin q, 0, -l cos q): U = -m g l cos q, dU/dq = m g l sin q
    assert abs(d["h"][0, 0] - m * G * l * np.sin(q)) < 1e-12


@pytest.mark.parametrize("which", ["anymal", "pendulum", "atlas", *INSTANCE_MODELS])
def test_gravity_bias_is_potential_gradient(which, anymal_tables, atlas_tables):
    t = _tables(which, anymal_tables, atlas_tables)
    o = Oracle(t)
    rng = np.random.default_rng(2)
    gc, gv = random_state(t, rng, 2, vel_scale=0.0)
    gc0 = gc.copy()
    d = o.step(gc, gv, n_steps=1, debug=True)
    eps = 1e-6
    for e in range(2):
        grad = np.zeros(t["nv"])
        for k in range(t["nv"]):
            dv = np.zeros(t["nv"]); dv[k] = 1.0
            grad[k] = (potential_energy(t, integrate_gc(t, gc0[e], dv, eps)) - potential_energy(t, integrate_gc(t, gc0[e], dv, -eps))) / (2 * eps)
        assert np.allclose(d["h"][e], grad, atol=2e-5 * max(1.0, np.abs(grad).max()))


@pytest.mark.parametrize("which", ["anymal", "pendulum", "atlas", *INSTANCE_MODELS])
def test_coriolis_bias_vs_lagrangian(which, anymal_tables, atlas_tables):
    """h(q,v) - h(q,0) must equal Mdot v - 1/2 d(v^T M v)/dq, with M from the independent numpy
    restatement and derivatives by central differences along the oracle's own (+) operator."""
    t = _tables(which, anymal_tables, atlas_tables)
    o = Oracle(t, params=dict(gx=0.0, gy=0.0, gz=0.0))
    rng = np.random.default_rng(3)
    gc, gv = random_state(t, rng, 1, vel_scale=1.0)
    q0, v0 = gc[0].copy(), gv[0].copy()
    d = o.step(gc, gv, n_steps=1, debug=True)
    eps = 1e-5
    nv = t["nv"]
    Mdot = (mass_matrix_numpy(t, integrate_gc(t, q0, v0, eps)) - mass_matrix_numpy(t, integrate_gc(t, q0, v0, -eps))) / (2 * eps)
    dT = np.zeros(nv)
    for k in range(nv):
        dv = np.zeros(nv); dv[k] = 1.0
        Mp, Mm = mass_matrix_numpy(t, integrate_gc(t, q0, dv, eps)), mass_matrix_numpy(t, integrate_gc(t, q0, dv, -eps))
        dT[k] = 0.5 * v0 @ (Mp - Mm) @ v0 / (2 * eps)
    c_ref = Mdot @ v0 - dT
    if t["floating"]:
        # quasi-velocity correction for the world-frame angular velocity of the base:
        # d/dt(dT/dw) - (dT/dphi) picks up  w x (dT/dw) ... handled by comparing joint rows and the
        # linear rows only (those use true coordinates); rotational rows are checked through the
        # energy / momentum tests below.
        rows = np.r_[0:3, 6:nv]
    else:
        rows = np.arange(nv)
    scale = max(1.0, np.abs(c_ref).max())
    assert np.allclose(d["h"][0][rows], c_ref[rows], atol=2e-4 * scale)


@pytest.mark.parametrize("which", ["anymal", "atlas"])
def test_energy_and_momentum_conservation_zero_g(which, anymal_tables, atlas_tables):
    t = {"anymal": anymal_tables, "atlas": atlas_tables}[which]
    dt = 1e-4
    o = Oracle(t, params=dict(gz=0.0, dt=dt))
    rng = np.random.default_rng(4)
    gc, gv = random_state(t, rng, 1, vel_scale=0.5)

    def invariants(q, v):
        M = mass_matrix_numpy(t, q)
        P = M[0:3] @ v
        Lo = M[3:6] @ v                     # angular momentum about the base origin
        return 0.5 * v @ M @ v, P, Lo + np.cross(q[0:3], P)

    E0, P0, L0 = invariants(gc[0], gv[0])
    o.step(gc, gv, n_steps=200)
    E1, P1, L1 = invariants(gc[0], gv[0])
    assert np.allclose(P1, P0, atol=1e-9 * max(1, np.abs(P0).max()))       # exact for this integrator
    assert np.allclose(L1, L0, rtol=0, atol=2e-3 * np.abs(L0).max())        # O(dt) drift
    assert abs(E1 - E0) < 2e-3 * E0


def test_sphere_rest_on_plane():
    t = load_tables(SPHERE_URDF)
    o = Oracle(t)
    o.set_ground(0.0)
    gc = np.array([[0, 0, 0.0999, 1, 0, 0, 0.0]]); gv = np.zeros((1, 6))
    d = o.step(gc, gv, n_steps=1, debug=True)
    assert d["ncontacts"][0] == 1 and d["c_pair"][0, 0] == 0 and d["c_body"][0, 0] == 0
    assert np.allclose(d["c_lambda"][0, 0], [0, 0, 2.0 * G * 0.0025], atol=1e-9)
    assert np.allclose(gv[0], 0, atol=1e-9)
    assert abs(d["c_depth"][0, 0] - 1e-4) < 1e-12
    # ERP pushes the penetration out: v_n+ = erp * depth / dt
    o.set_params(erp=0.2)
    gc = np.array([[0, 0, 0.0999, 1, 0, 0, 0.0]]); gv = np.zeros((1, 6))
    o.step(gc, gv, n_steps=1)
    assert abs(gv[0, 2] - 0.2 * 1e-4 / 0.0025) < 1e-9


def test_sphere_restitution():
    t = load_tables(SPHERE_URDF)
    o = Oracle(t, params=dict(restitution=0.5, gz=0.0))
    o.set_ground(0.0)
    gc = np.array([[0, 0, 0.0999, 1, 0, 0, 0.0]]); gv = np.zeros((1, 6)); gv[0, 2] = -1.0
    o.step(gc, gv, n_steps=1)
    assert abs(gv[0, 2] - 0.5) < 1e-9


@pytest.mark.parametrize("slope_deg,expect_slide", [(20.0, False), (35.0, False), (42.0, True), (60.0, True)])
def test_box_on_slope_stick_slip_threshold(slope_deg, expect_slide):
    """Tilt gravity instead of the plane.  mu = 0.8 -> threshold atan(0.8) = 38.66 deg."""
    t = load_tables(BOX_URDF)
    th = np.deg2rad(slope_deg)
    o = Oracle(t, params=dict(gx=G * np.sin(th), gz=-G * np.cos(th), mu=0.8))
    o.set_ground(0.0)
    gc = np.array([[0, 0, 0.0999, 1, 0, 0, 0.0]]); gv = np.zeros((1, 6))
    n, dt = 100, 0.0025
    d = o.step(gc, gv, n_steps=n, debug=True)
    assert d["ncontacts"][0] == 4
    if expect_slide:
        lam = d["c_lambda"][0, :4]
        # slip: every contact on the cone surface, friction opposes the motion
        assert np.allclose(np.hypot(lam[:, 0], lam[:, 1]), 0.8 * lam[:, 2], rtol=1e-5)
        assert (lam[:, 0] < 0).all()
        assert abs(lam[:, 2].sum() - 3.0 * G * np.cos(th) * dt) < 1e-9
        # the per-contact rule dissipates in each contact's own apparent-inertia metric (Hwangbo 2018
        # eq. for the slip case), so with normal-tangential coupling (box corners) the lateral
        # components cancel pairwise and the net friction is slightly below mu * sum(lambda_n)
        fx = -lam[:, 0].sum()
        assert 0.95 * 0.8 * lam[:, 2].sum() < fx <= 0.8 * lam[:, 2].sum() + 1e-12
        assert abs(lam[:, 1].sum()) < 1e-9
        acc = G * np.sin(th) - fx / (3.0 * dt)
        assert abs(gv[0, 0] - acc * n * dt) < 1e-6
    else:
        assert np.abs(gv[0]).max() < 1e-6
    assert abs(gv[0, 2]) < 1e-6


def test_sliding_sphere_exact_coulomb():
    """Single sphere contact: the normal passes through the COM, no normal-tangential coupling,
    so the slip impulse opposes the sliding velocity exactly with magnitude mu * lambda_n."""
    t = load_tables(SPHERE_URDF)
    o = Oracle(t, params=dict(mu=0.5))
    o.set_ground(0.0)
    gc = np.array([[0, 0, 0.0999, 1, 0, 0, 0.0]]); gv = np.zeros((1, 6)); gv[0, 0] = 3.0; gv[0, 1] = -4.0
    dt, m, r, I = 0.0025, 2.0, 0.1, 0.008
    d = o.step(gc, gv, n_steps=1, debug=True)
    lam = d["c_lambda"][0, 0]
    assert abs(lam[2] - m * G * dt) < 1e-9
    assert np.allclose(lam[:2], -0.5 * lam[2] * np.array([3.0, -4.0]) / 5.0, atol=1e-8)
    assert np.allclose(gv[0, :2], (1 - 0.5 * G * dt / 5.0) * np.array([3.0, -4.0]), atol=1e-8)
    # the friction impulse spins the ball up about the axis n x f
    w_expected = np.cross(np.array([0, 0, -r]), np.array([lam[0], lam[1], 0.0])) / I
    assert np.allclose(gv[0, 3:6], w_expected, atol=1e-7)


def test_sliding_friction_decelerates_then_sticks():
    t = load_tables(BOX_URDF)
    o = Oracle(t)
    o.set_ground(0.0)
    gc = np.array([[0, 0, 0.0999, 1, 0, 0, 0.0]]); gv = np.zeros((1, 6)); gv[0, 0] = 1.0; gv[0, 1] = 0.5
    dt = 0.0025
    v0 = gv[0, :2].copy()
    o.step(gc, gv, n_steps=20)
    # deceleration mu*g along the motion direction (centre of mass above the contacts adds a small
    # pitching couple; the box is flat enough to stay down)
    speed = np.linalg.norm(gv[0, :2])
    assert 0.95 * 0.8 * G * 20 * dt < np.linalg.norm(v0) - speed <= 0.8 * G * 20 * dt + 1e-9
    assert abs(np.cross(gv[0, :2], v0)) < 2e-2      # direction (nearly) preserved
    o.step(gc, gv, n_steps=200)
    assert np.abs(gv[0]).max() < 1e-6               # came to rest and stays


def _f_energy(Gm, c, lam):
    return c @ lam + 0.5 * lam @ Gm @ lam


def test_per_contact_solver_against_dense_scan(anymal_tables):
    """solve_one (stick / slip / open) against a brute-force scan of the cone-surface x zero-normal-
    velocity curve (Hwangbo et al. 2018 section IV)."""
    o = Oracle(anymal_tables)
    rng = np.random.default_rng(7)
    n_slip = 0
    for trial in range(300):
        A = rng.standard_normal((3, 5))
        Gm = A @ A.T * 0.02 + 0.01 * np.eye(3)
        c = rng.standard_normal(3) * np.array([1.0, 1.0, 0.5])
        mu = rng.uniform(0.2, 1.2)
        lam = o.solve_one(Gm, c, mu)
        if c[2] > 0:
            assert np.allclose(lam, 0)
            continue
        ls = -np.linalg.solve(Gm, c)
        if ls[2] >= 0 and np.hypot(ls[0], ls[1]) <= mu * ls[2]:
            assert np.allclose(lam, ls, rtol=1e-9, atol=1e-12)
            continue
        th = np.linspace(0, 2 * np.pi, 20001)
        D = Gm[2, 2] + mu * (Gm[2, 0] * np.cos(th) + Gm[2, 1] * np.sin(th))
        if (D <= 1e-9).any():
            continue
        n_slip += 1
        lz = -c[2] / D
        L = np.stack([mu * lz * np.cos(th), mu * lz * np.sin(th), lz], 1)
        f = L @ c + 0.5 * np.einsum("ij,jk,ik->i", L, Gm, L)
        fmin = f.min()
        v = c + Gm @ lam
        assert abs(v[2]) < 1e-9 * max(1, np.abs(c).max())             # zero normal velocity
        assert abs(np.hypot(lam[0], lam[1]) - mu * lam[2]) < 1e-9      # on the cone surface
        assert lam[2] >= 0
        # a local minimum of the energy on the curve, no worse than the global scan by more than the scan step
        fl = _f_energy(Gm, c, lam)
        tl = np.arctan2(lam[1], lam[0])
        for dth in (-1e-4, 1e-4):
            Dn = Gm[2, 2] + mu * (Gm[2, 0] * np.cos(tl + dth) + Gm[2, 1] * np.sin(tl + dth))
            ln = (-c[2] / Dn) * np.array([mu * np.cos(tl + dth), mu * np.sin(tl + dth), 1.0])
            assert _f_energy(Gm, c, ln) >= fl - 1e-12
        assert fl <= fmin + 1e-6 * max(1.0, abs(fmin))
    assert n_slip > 50


def test_solver_f32_matches_f64(anymal_tables):
    o64, o32 = Oracle(anymal_tables), Oracle(anymal_tables, precision="f32")
    rng = np.random.default_rng(8)
    for trial in range(200):
        A = rng.standard_normal((3, 5))
        Gm = (A @ A.T * 0.02 + 0.01 * np.eye(3)).astype(np.float32).astype(np.float64)
        c = rng.standard_normal(3).astype(np.float32).astype(np.float64)
        a, b = o64.solve_one(Gm, c, 0.8), o32.solve_one(Gm, c, 0.8)
        assert np.allclose(a, b, rtol=2e-4, atol=2e-5 * max(1, np.abs(a).max()))


def test_complementarity_after_solve(anymal_tables):
    """Signorini + Coulomb residuals on a contact-rich random batch (robots dropped in random poses)."""
    t = anymal_tables
    o = Oracle(t, params=dict(threshold=1e-10, max_iter=500, stall_window=0))
    o.set_ground(0.0)
    rng = np.random.default_rng(9)
    gc, gv = random_state(t, rng, 64, vel_scale=0.5, base_z=0.35)
    seen_contacts = 0
    for it in range(40):
        q_before, v_before = gc.copy(), gv.copy()
        d = o.step(gc, gv, n_steps=1, debug=True)
        for e in range(64):
            K = d["ncontacts"][e]
            seen_contacts += K
            if K == 0 or d["iters"][e] >= 500:
                continue
            lam = d["c_lambda"][e, :K]
            assert (lam[:, 2] >= -1e-12).all()
            assert (np.hypot(lam[:, 0], lam[:, 1]) <= 0.8 * lam[:, 2] + 1e-7).all()
            # post-step normal velocity of every contact point, recomputed independently from v+
            bj = body_jacobians(t, q_before[e])
            R, p, a = fk_numpy(t, q_before[e])
            for k in range(K):
                b, pos, n = d["c_body"][e, k], d["c_pos"][e, k], d["c_normal"][e, k]
                J = np.zeros((3, t["nv"]))
                J[:, 0:3] = np.eye(3)
                r = pos - p[0]
                J[:, 3:6] = -np.array([[0, -r[2], r[1]], [r[2], 0, -r[0]], [-r[1], r[0], 0]])
                j = b
                while t["parent"][j] >= 0:
                    J[:, t["vidx"][j]] = np.cross(a[j], pos - p[j])
                    j = t["parent"][j]
                vn = n @ (J @ gv[e])
                assert vn >= -1e-6
                assert abs(vn * lam[k, 2]) < 1e-6
    assert seen_contacts > 1000


def test_heightmap_flat_equals_ground(anymal_tables):
    t = anymal_tables
    o1, o2 = Oracle(t), Oracle(t)
    o1.set_ground(0.05)
    o2.set_heightmap(17, 9, 8.0, 4.0, 0.3, -0.2, np.full(17 * 9, 0.05))
    rng = np.random.default_rng(10)
    gc, gv = random_state(t, rng, 16, vel_scale=0.5, base_z=0.4, pos_scale=1.0)
    gca, gva, gcb, gvb = gc.copy(), gv.copy(), gc.copy(), gv.copy()
    da = o1.step(gca, gva, n_steps=20, debug=True)
    db = o2.step(gcb, gvb, n_steps=20, debug=True)
    assert (da["ncontacts"] == db["ncontacts"]).all() and da["ncontacts"].sum() > 0
    assert (da["c_pt"] == db["c_pt"]).all()
    assert np.allclose(gca, gcb, atol=1e-9) and np.allclose(gva, gvb, atol=1e-8)


def test_heightmap_tilted_plane_normal_and_depth():
    t = load_tables(SPHERE_URDF)
    o = Oracle(t)
    xs, ys, X, Y = 11, 11, 10.0, 10.0
    gx = np.linspace(-5, 5, xs); gy = np.linspace(-5, 5, ys)
    H = 0.3 * gx[None, :] + 0.1 * gy[:, None]          # z = 0.3 x + 0.1 y, h[iy*xs+ix]
    o.set_heightmap(xs, ys, X, Y, 0.0, 0.0, H)
    n = np.array([-0.3, -0.1, 1.0]); n /= np.linalg.norm(n)
    P = np.array([1.23, -0.57, 0.0]); P[2] = 0.3 * P[0] + 0.1 * P[1]
    centre = P + n * (0.1 - 0.002)                      # sphere r=0.1 penetrating 2 mm along the normal
    gc = np.array([[*centre, 1, 0, 0, 0.0]]); gv = np.zeros((1, 6))
    d = o.step(gc, gv, n_steps=1, debug=True)
    assert d["ncontacts"][0] == 1
    assert np.allclose(d["c_normal"][0, 0], n, atol=1e-12)
    assert abs(d["c_depth"][0, 0] - 0.002) < 1e-12
    ix, iy = int((P[0] + 5) / 1.0), int((P[1] + 5) / 1.0)        # the triangle that holds the touched point
    fx, fy = (P[0] + 5) - ix, (P[1] + 5) - iy
    assert d["c_pair"][0, 0] == 2 * (iy * (xs - 1) + ix) + (0 if fx >= fy else 1)
    # outside the map: no contact
    gc = np.array([[7.0, 0, -3.0, 1, 0, 0, 0.0]])
    d = o.step(gc, np.zeros((1, 6)), n_steps=1, debug=True)
    assert d["ncontacts"][0] == 0


def test_contact_cap_keeps_deepest(atlas_tables):
    t = atlas_tables
    o = Oracle(t)
    o.set_ground(0.0)
    gc = np.zeros((1, 37)); gc[0, 2] = 0.05; gc[0, 3:7] = [np.cos(np.pi / 4), 0, np.sin(np.pi / 4), 0]   # lying face down
    gv = np.zeros((1, 36))
    d = o.step(gc, gv, n_steps=1, debug=True)
    assert d["ncontacts"][0] == o.kmax
    pts = d["c_pt"][0]
    assert (np.diff(pts) > 0).all()


def test_pd_implicit_stability(anymal_tables):
    """Stiff PD (kp*dt^2 >> joint inertia) must stay bounded thanks to the implicit treatment."""
    t = anymal_tables
    o = Oracle(t, params=dict(gz=0.0))
    gc = ANYMAL_GC0[None].copy(); gc[0, 2] = 5.0
    gv = np.zeros((1, 18))
    target = ANYMAL_GC0[None].copy(); target[0, 7:] += 0.3
    kp = np.r_[np.zeros(6), 1e5 * np.ones(12)]; kd = np.r_[np.zeros(6), 10.0 * np.ones(12)]
    o.step(gc, gv, n_steps=400, ptarget=target, kp=kp, kd=kd)
    assert np.isfinite(gc).all()
    assert np.allclose(gc[0, 7:], target[0, 7:], atol=2e-2)


def test_stagnation_exit_only_hits_cycling_problems(anymal_tables):
    """stall_window (include/rsb.h): converged environments are untouched, cycling ones stop early."""
    t = anymal_tables
    rng = np.random.default_rng(12)
    gc, gv = random_state(t, rng, 256, vel_scale=0.5, base_z=0.35)
    res = {}
    for w in (0, 8):
        o = Oracle(t, params=dict(threshold=1e-6, stall_window=w))
        o.set_ground(0.0)
        a, b = gc.copy(), gv.copy()
        d = o.step(a, b, n_steps=1, debug=True)
        res[w] = (a, b, d["iters"].copy(), d["status"].copy())
    it0, it8 = res[0][2], res[8][2]
    conv = it0 < 150
    untouched = it8[conv] == it0[conv]
    # environments that converge within the first two windows can never be cut short ...
    assert (it8[conv & (it0 <= 16)] == it0[conv & (it0 <= 16)]).all()
    assert np.array_equal(res[0][1][conv & (it0 <= 16)], res[8][1][conv & (it0 <= 16)])
    # ... slow (> 16 iterations) convergers may be (measured: ~11 % of this deliberately brutal batch of
    # robots dropped in random orientations half inside the ground; 0 of 600 in a kneeling-robot batch)
    assert untouched.mean() > 0.85
    # cycling cases: the first failed check switches to the compliant contact set (stall_reg), on which most of them converge;
    # a second failed check ends the rest -- well before max_iter either way
    st8 = res[8][3]
    assert (~conv).sum() > 0 and it8[~conv].max() <= 110
    assert (st8[~conv] == 1).mean() >= 0.5 and set(np.unique(st8)) <= {0, 1, 2}
    assert (res[0][3][~conv] == 3).all() and (res[0][3][conv] == 0).all()      # without the check: max_iter


def test_bisection_and_32_section_slip_search_agree(anymal_tables):
    """slip_bisect=1 (CPU-tuned search used for the CPU baseline timing) vs the kernel-identical 32-section rounds"""
    oa, ob = Oracle(anymal_tables), Oracle(anymal_tables, params=dict(slip_bisect=1))
    rng = np.random.default_rng(15)
    n_slip = 0
    for trial in range(300):
        A = rng.standard_normal((3, 5))
        Gm = A @ A.T * 0.02 + 0.01 * np.eye(3)
        c = rng.standard_normal(3) * np.array([1.0, 1.0, 0.5])
        mu = rng.uniform(0.2, 1.2)
        la, lb = oa.solve_one(Gm, c, mu), ob.solve_one(Gm, c, mu)
        # two regula-falsi steps from a 6e-3 rad bracket vs ten halvings + a secant step: the same root to ~1e-6 of the impulse
        assert np.allclose(la, lb, rtol=5e-6, atol=5e-6 * max(1.0, np.abs(la).max()))
        n_slip += int(c[2] <= 0 and abs(np.hypot(la[0], la[1]) - mu * la[2]) < 1e-9 and la[2] > 0)
    assert n_slip > 50
    t = anymal_tables
    gc, gv = random_state(t, np.random.default_rng(16), 64, vel_scale=0.5, base_z=0.5)
    outs = []
    for o in (Oracle(t, params=dict(threshold=1e-8, stall_window=0)), Oracle(t, params=dict(threshold=1e-8, stall_window=0, slip_bisect=1))):
        o.set_ground(0.0)
        a, b = gc.copy(), gv.copy()
        d = o.step(a, b, n_steps=5, debug=True)
        outs.append((a, b, d["iters"]))
    conv = (outs[0][2] < 150) & (outs[1][2] < 150)
    assert np.abs(outs[0][1] - outs[1][1])[conv].max() < 1e-5


LIMIT_PENDULUM = """<robot name="p"><link name="world"/>
  <link name="l"><inertial><origin xyz="0 0 -0.5"/><mass value="2.0"/><inertia ixx="0.1" ixy="0" ixz="0" iyy="0.1" iyz="0" izz="0.01"/></inertial></link>
  <joint name="j" type="revolute"><parent link="world"/><child link="l"/><origin xyz="0 0 1"/><axis xyz="0 1 0"/>
    <limit lower="-0.5" upper="0.5" effort="10" velocity="10"/></joint></robot>"""


def test_joint_limit_stops_motion_inelastically():
    t = load_tables(LIMIT_PENDULUM)
    o = Oracle(t, params=dict(gz=0.0))
    gc, gv = np.array([[0.45]]), np.array([[2.0]])
    qs = []
    for k in range(40):
        d = o.step(gc, gv, n_steps=1, debug=True)
        qs.append(gc[0, 0])
    assert max(qs) <= 0.5 + 2.0 * 0.0025 + 1e-12        # at most one step of overshoot
    assert abs(gv[0, 0]) < 1e-12 and d["nlimits"][0] == 1 and d["lim_dof"][0, 0] == 0
    # ERP turns the overshoot into an inward velocity erp * viol / dt; the row releases once the joint is back inside
    q_over = gc[0, 0]
    o.set_params(erp=0.2)
    o.step(gc, gv, n_steps=1)
    assert abs(gv[0, 0] + 0.2 * (q_over - 0.5) / 0.0025) < 1e-9
    o.step(gc, gv, n_steps=100)
    assert gc[0, 0] < 0.5 and gv[0, 0] < 0
    # switched off: the joint sails through
    o2 = Oracle(t, params=dict(gz=0.0, joint_limits=0))
    gc, gv = np.array([[0.45]]), np.array([[2.0]])
    o2.step(gc, gv, n_steps=40)
    assert gc[0, 0] > 0.6


def test_joint_limit_reaction_balances_gravity():
    t = load_tables(LIMIT_PENDULUM)
    o = Oracle(t)
    q0 = 0.5004                                          # resting just beyond the upper stop, gravity pulls it back? no: push it out
    o.set_params(gx=3.0)                                 # a sideways "gravity" component presses the link against the stop
    gc, gv = np.array([[q0]]), np.array([[0.0]])
    d = o.step(gc, gv, n_steps=1, debug=True)
    m, l, I, dt = 2.0, 0.5, 0.1, 0.0025
    # generalized force of gravity about +y at angle q: COM at (-l sin q, 0, -l cos q)
    tau_g = m * (3.0 * (-l * np.cos(q0)) - (-9.81) * (-l * np.sin(q0)))
    if tau_g > 0:                                        # gravity drives q further past the stop: the stop must hold it
        assert d["nlimits"][0] == 1
        assert abs(d["lim_lambda"][0, 0] - tau_g * dt) < 1e-9
        assert abs(gv[0, 0]) < 1e-12
    else:                                                # gravity pulls it back inside: the row stays passive
        assert abs(d["lim_lambda"][0, 0]) < 1e-15 and gv[0, 0] < 0


def test_joint_limit_is_internal_momentum_conserved(anymal_tables):
    """a limit impulse is an internal generalized force: total momentum of the free-floating robot is unchanged"""
    t = anymal_tables
    o = Oracle(t, params=dict(gz=0.0, dt=1e-3))
    gc = ANYMAL_GC0[None].copy(); gc[0, 2] = 5.0
    gc[0, 7] = 0.49 - 1e-4                               # LF_HAA just inside its upper stop (0.49)
    gv = np.zeros((1, 18)); gv[0, 6] = 3.0               # swinging into it
    M0 = mass_matrix_numpy(t, gc[0]); P0, L0 = M0[0:3] @ gv[0], M0[3:6] @ gv[0] + np.cross(gc[0, 0:3], M0[0:3] @ gv[0])
    hit = 0
    for k in range(30):
        d = o.step(gc, gv, n_steps=1, debug=True)
        hit += int(d["nlimits"][0] > 0 and d["lim_lambda"][0, 0] > 0)
    M1 = mass_matrix_numpy(t, gc[0]); P1, L1 = M1[0:3] @ gv[0], M1[3:6] @ gv[0] + np.cross(gc[0, 0:3], M1[0:3] @ gv[0])
    assert hit >= 1
    assert gc[0, 7] < 0.49 + 3.0 * 1e-3 + 1e-9           # stopped within one step of overshoot
    # an impulsive stop changes v by 3 rad/s inside one step while the bias force was evaluated with the pre-impact
    # velocity: the discrete momentum error of that single step is O(dt * |h|) ~ 6e-3, then it stays constant
    assert np.allclose(P1, P0, atol=1e-2) and np.allclose(L1, L0, atol=1e-2 * np.abs(L0).max() + 1e-6)


def test_per_body_friction_override():
    """a low-friction collision body slides where the default material sticks (World::setMaterialPairProp analogue)"""
    t = load_tables(BOX_URDF)
    th = np.deg2rad(20.0)                                # tan 20 deg = 0.364: sticks at mu 0.8, slides at mu 0.2
    res = {}
    for mu in (-1.0, 0.2):
        o = Oracle(t, params=dict(gx=G * np.sin(th), gz=-G * np.cos(th)))
        o.set_ground(0.0)
        o.set_collision_friction(0, mu)
        gc = np.array([[0, 0, 0.0999, 1, 0, 0, 0.0]]); gv = np.zeros((1, 6))
        o.step(gc, gv, n_steps=100)
        res[mu] = gv[0, 0]
    assert abs(res[-1.0]) < 1e-6
    acc = G * (np.sin(th) - 0.2 * np.cos(th))
    assert 0.9 * acc * 0.25 < res[0.2] <= 1.08 * acc * 0.25


@pytest.mark.parametrize("which", ["anymal", "atlas"])
def test_external_wrench_momentum_balance(which, anymal_tables, atlas_tables):
    """setExternalForce / setExternalTorque: over one step in zero gravity the free-floating robot's linear momentum
    changes by F dt and its angular momentum about the world origin by (r x F + T) dt, wherever the wrench acts."""
    t = {"anymal": anymal_tables, "atlas": atlas_tables}[which]
    dt = 1e-4
    o = Oracle(t, params=dict(gz=0.0, dt=dt))
    rng = np.random.default_rng(14)
    gc, gv = random_state(t, rng, 1, vel_scale=0.3)
    body = t["nb"] - 1                                # a distal link
    F, T, pb = np.array([3.0, -2.0, 5.0]), np.array([0.4, 0.1, -0.3]), np.array([0.05, -0.02, 0.1])

    def momenta(q, v):
        M = mass_matrix_numpy(t, q)
        P = M[0:3] @ v
        return P, M[3:6] @ v + np.cross(q[0:3], P)

    R, p, _a = fk_numpy(t, gc[0])
    r_world = p[body] + R[body] @ pb
    P0, L0 = momenta(gc[0], gv[0])
    q0, gv_before = gc.copy(), gv.copy()
    o.step(gc, gv, n_steps=1, ext=(body, F, T, pb))
    P1, L1 = momenta(q0[0], gv[0])                     # same configuration: isolates the velocity change of the step
    # the same step without the wrench gives the baseline (the integrator's own O(dt) change of L is common to both)
    gcb, gvb = q0.copy(), gv_before.copy()
    o.step(gcb, gvb, n_steps=1)
    Pb, Lb = momenta(q0[0], gvb[0])
    assert np.allclose(P1 - Pb, F * dt, atol=1e-9)
    assert np.allclose(L1 - Lb, (np.cross(r_world, F) + T) * dt, atol=1e-9)


def test_external_torque_on_pendulum_closed_form():
    urdf = """<robot name="p"><link name="world"/>
      <link name="l"><inertial><origin xyz="0 0 -0.5"/><mass value="2.0"/><inertia ixx="0.1" ixy="0" ixz="0" iyy="0.1" iyz="0" izz="0.01"/></inertial></link>
      <joint name="j" type="revolute"><parent link="world"/><child link="l"/><origin xyz="0 0 1"/><axis xyz="0 1 0"/></joint></robot>"""
    t = load_tables(urdf)
    dt = 1e-3
    o = Oracle(t, params=dict(gz=0.0, dt=dt))
    m, l, I = 2.0, 0.5, 0.1
    gc, gv = np.array([[0.0]]), np.array([[0.0]])
    o.step(gc, gv, ext=(1, None, np.array([0.0, 0.7, 0.0]), None))          # pure torque about the joint axis
    assert abs(gv[0, 0] - 0.7 * dt / (I + m * l * l)) < 1e-12
    gc, gv = np.array([[0.0]]), np.array([[0.0]])
    o.step(gc, gv, ext=(1, np.array([1.5, 0.0, 0.0]), None, np.array([0.0, 0.0, -1.0])))   # force at 1 m below the pivot
    # rotation about +y: x-velocity of a point at z = -1 is -qdot, so the generalized force is -1.5 * 1
    assert abs(gv[0, 0] - (-1.5 * dt / (I + m * l * l))) < 1e-12
    gc, gv = np.array([[0.0]]), np.array([[0.0]])
    o.step(gc, gv)                                                            # the wrench does not persist
    assert gv[0, 0] == 0.0


def test_flop_counting_build_matches_f64_and_reports_algorithmic_flops(anymal_tables):
    """SURVEY 8(d): ALGORITHMIC FLOPs per env-step counted with an instrumented scalar (Sim<Cnt>); the counting build is
    the float64 restatement operation for operation, so its results are bit-identical."""
    from oracle.oracle import flop_counters
    t = anymal_tables
    n = 32
    rng = np.random.default_rng(77)
    gc = np.tile(ANYMAL_GC0, (n, 1)); gc[:, 2] = 0.58; gc[:, 7:] += rng.uniform(-0.1, 0.1, (n, 12))
    gv = np.zeros((n, 18))
    kp = np.r_[np.zeros(6), 300.0 * np.ones(12)]; kd = np.r_[np.zeros(6), 8.0 * np.ones(12)]
    tgt = np.tile(ANYMAL_GC0, (n, 1))
    o = Oracle(t, params=dict(threshold=1e-6)); oc = Oracle(t, precision="count", params=dict(threshold=1e-6))
    for x in (o, oc):
        x.set_ground(0.0)
    o.step(gc, gv, n_steps=200, ptarget=tgt, vtarget=np.zeros((n, 18)), kp=kp, kd=kd)       # settle on the ground
    a, b = gc.copy(), gv.copy()
    flop_counters()
    d = oc.step(a, b, n_steps=4, ptarget=tgt, vtarget=np.zeros((n, 18)), kp=kp, kd=kd, debug=True)
    c = flop_counters()
    o.step(gc, gv, n_steps=4, ptarget=tgt, vtarget=np.zeros((n, 18)), kp=kp, kd=kd)
    assert np.array_equal(a, gc) and np.array_equal(b, gv)
    flops = (c["add"] + c["mul"] + c["div"] + c["sqrt"]) / (4 * n)
    print(f"algorithmic FLOPs per env-step (dense restatement, K mean {d['ncontacts'].mean():.2f}): {flops:.0f}  {c}")
    assert d["ncontacts"].mean() > 3.5 and 20e3 < flops < 80e3           # SURVEY 8(d) estimated 30-60 k for ANYmal with K = 4


def test_terrain_atlas_gives_every_environment_its_own_map():
    """N3: per-environment height maps.  Flat maps at different heights: a resting sphere ends up on ITS map."""
    t = load_tables(SPHERE_URDF)
    o = Oracle(t, params=dict(dt=0.002))
    n, xs, ys = 6, 9, 7
    levels = np.array([0.0, 0.25, -0.1])
    H = np.tile(levels[:, None, None], (1, ys, xs))
    env_map = np.array([0, 1, 2, 2, 1, 0], np.int32)
    o.set_heightmaps(4.0, 3.0, 0.0, 0.0, H, env_map)
    gc = np.zeros((n, 7)); gc[:, 3] = 1.0; gc[:, 2] = levels[env_map] + 0.1 + 0.05      # sphere radius 0.1: 5 cm above its own map
    gv = np.zeros((n, 6))
    o.step(gc, gv, n_steps=400)
    assert np.allclose(gc[:, 2], levels[env_map] + 0.1, atol=2e-3)
    # identical maps in the atlas == the single-map call
    rng = np.random.default_rng(2)
    Hr = 0.05 * rng.uniform(-1, 1, (ys, xs))
    a, b = np.zeros((n, 7)), np.zeros((n, 6)); a[:, 3] = 1.0; a[:, 2] = 0.12; a[:, 0] = np.linspace(-1, 1, n)
    c, d = a.copy(), b.copy()
    o.set_heightmaps(4.0, 3.0, 0.0, 0.0, np.stack([Hr, Hr]), np.array([0, 1, 0, 1, 1, 0], np.int32))
    o.step(a, b, n_steps=50)
    o.set_heightmap(xs, ys, 4.0, 3.0, 0.0, 0.0, Hr)
    o.step(c, d, n_steps=50)
    assert np.array_equal(a, c) and np.array_equal(b, d)


def test_anderson_accelerated_gauss_seidel_same_fixed_point_fewer_sweeps(atlas_tables):
    """Anderson acceleration of the Gauss-Seidel sweep map (accel_m = 2 by default in oracle and kernel; DESIGN.md section 5).
    Redundant box-corner contacts of the standing humanoid: same solution, a third of the sweeps."""
    t = atlas_tables
    n = 64
    rng = np.random.default_rng(3)
    gc = np.zeros((n, 37)); gc[:, 2] = 0.95; gc[:, 3] = 1.0; gc[:, 7:] += rng.uniform(-0.05, 0.05, (n, 30))
    gv = np.zeros((n, 36))
    kp = np.r_[np.zeros(6), 400 * np.ones(30)]; kd = np.r_[np.zeros(6), 10 * np.ones(30)]
    tgt = gc.copy()
    plain = Oracle(t, params=dict(threshold=1e-7, stall_window=0, accel_m=0)); plain.set_ground(0.0)
    plain.step(gc, gv, n_steps=60, ptarget=tgt, vtarget=np.zeros((n, 36)), kp=kp, kd=kd)          # settle onto the feet
    acc = Oracle(t, params=dict(threshold=1e-7, stall_window=0, accel_m=2)); acc.set_ground(0.0)
    a, b = gc.copy(), gv.copy(); c, d = gc.copy(), gv.copy()
    dp = plain.step(a, b, ptarget=tgt, vtarget=np.zeros((n, 36)), kp=kp, kd=kd, debug=True)
    da = acc.step(c, d, ptarget=tgt, vtarget=np.zeros((n, 36)), kp=kp, kd=kd, debug=True)
    both = (dp["iters"] < 150) & (da["iters"] < 150)
    assert both.mean() > 0.9 and (dp["ncontacts"] >= 6).mean() > 0.9
    print(f"sweeps plain {dp['iters'][both].mean():.1f} accelerated {da['iters'][both].mean():.1f}; |dgv| {np.abs(b - d)[both].max():.2e}")
    assert da["iters"][both].mean() < 0.5 * dp["iters"][both].mean()
    assert np.abs(b - d)[both].max() < 2e-5          # same fixed point (velocity level), to the solver threshold
    # default parameters leave quickly converging problems untouched (acceleration starts at sweep 6)
    t2 = load_tables(SPHERE_URDF)
    o1, o2 = Oracle(t2, params=dict(accel_m=0)), Oracle(t2, params=dict(accel_m=2))
    for o in (o1, o2):
        o.set_ground(0.0)
    g1 = np.array([[0, 0, 0.1, 1, 0, 0, 0.0]]); v1 = np.array([[0.5, 0, -0.2, 0, 0, 0.0]]); g2, v2 = g1.copy(), v1.copy()
    o1.step(g1, v1, n_steps=20); o2.step(g2, v2, n_steps=20)
    assert np.array_equal(g1, g2) and np.array_equal(v1, v2)


# ---- a6 narrow phase against a HeightMap: shape vs every triangle under its bounding box (SURVEY 8c) ----------------------
def _single_shape_urdf(geometry, rpy="0 0 0"):
    return f"""<robot name="one"><link name="b"><inertial><origin xyz="0 0 0"/><mass value="2.0"/><inertia ixx="0.02" ixy="0" ixz="0" iyy="0.02" iyz="0" izz="0.02"/></inertial>
  <collision><origin xyz="0 0 0" rpy="{rpy}"/><geometry>{geometry}</geometry></collision></link></robot>"""


CAPSULE_X_URDF = _single_shape_urdf('<capsule radius="0.05" length="1.0"/>', rpy="0 1.5707963267948966 0")    # axis along world x
CYLINDER_Y_URDF = _single_shape_urdf('<cylinder radius="0.1" length="0.4"/>', rpy="1.5707963267948966 0 0")   # axis along world y
SPHERE5_URDF = _single_shape_urdf('<sphere radius="0.05"/>')


def ridge_map(n=21, pitch=0.1, top=0.3, slope=0.5):
    """a ridge along y at x = 0 (on a grid line): h = top - slope |x|"""
    x = (np.arange(n) - n // 2) * pitch
    return np.tile(top - slope * np.abs(x), (n, 1)), (n - 1) * pitch


def peak_map(n=21, pitch=0.1, h=0.2):
    H = np.zeros((n, n)); H[n // 2, n // 2] = h
    return H, (n - 1) * pitch


def _contacts_of(o, gc):
    gc = np.array([gc], float); gv = np.zeros((1, 6))
    d = o.step(gc, gv, debug=True)
    K = d["ncontacts"][0]
    return K, d["c_pt"][0][:K], d["c_pos"][0][:K], d["c_normal"][0][:K], d["c_depth"][0][:K], d["c_pair"][0][:K]


def test_capsule_lying_across_a_ridge_touches_with_its_side():
    """round 1 saw nothing here (two end spheres hanging in the air); the segment feature meets the ridge edge"""
    t = load_tables(CAPSULE_X_URDF)
    assert list(t["pt_type"]) == [0, 0, 1]
    H, size = ridge_map()
    o = Oracle(t); o.set_heightmap(21, 21, size, size, 0.0, 0.0, H)
    for cy, delta in ((0.03, 0.004), (0.27, 0.011), (-0.448, 0.002)):
        K, pt, pos, nrm, dep, pair = _contacts_of(o, [0.013, cy, 0.3 + 0.05 - delta, 1, 0, 0, 0])
        assert K == 1 and pt[0] == 2                                  # the segment candidate, not an end sphere
        assert abs(dep[0] - delta) < 1e-9 and np.allclose(nrm[0], [0, 0, 1], atol=1e-9)
        assert np.allclose(pos[0], [0.0, cy, 0.3 - delta], atol=1e-9)  # the capsule's surface point above the ridge line (contact positions are on the robot)
    # lifted clear of the ridge: nothing; tilted so that one end sphere digs into the slope: that end, not the side
    assert _contacts_of(o, [0.0, 0.0, 0.3 + 0.05 + 1e-4, 1, 0, 0, 0])[0] == 0
    K, pt, *_ = _contacts_of(o, [0.3, 0.0, 0.26, np.cos(0.35), 0, np.sin(0.35), 0])    # pitched: +x end down
    assert K >= 1 and (pt < 2).any()


def test_box_resting_on_a_peak_touches_with_its_face():
    t = load_tables(BOX_URDF)
    assert list(t["pt_type"]) == [0] * 8 + [2]
    H, size = peak_map()
    o = Oracle(t); o.set_heightmap(21, 21, size, size, 0.0, 0.0, H)
    delta = 0.007
    K, pt, pos, nrm, dep, pair = _contacts_of(o, [0.02, -0.01, 0.2 + 0.1 - delta, 1, 0, 0, 0])
    assert K == 1 and pt[0] == 8                                       # the eight corners hang over flat ground 0.2 m below
    assert abs(dep[0] - delta) < 1e-12 and np.allclose(nrm[0], [0, 0, 1]) and np.allclose(pos[0], [0, 0, 0.2])
    assert pair[0] == 2 * (10 * 20 + 10)                               # the cell whose lower-left vertex is the peak
    # rolled by 30 degrees about x: still the bottom face, the normal follows the box
    a = np.deg2rad(30.0)
    K, pt, pos, nrm, dep, pair = _contacts_of(o, [0.0, 0.0, 0.2 + (0.1 - delta) / np.cos(a), np.cos(a / 2), np.sin(a / 2), 0, 0])
    assert K == 1 and pt[0] == 8 and np.allclose(nrm[0], [0, -np.sin(a), np.cos(a)], atol=1e-9) and abs(dep[0] - delta) < 1e-9   # depth along the face normal


def test_sphere_on_a_ridge_and_in_a_valley_uses_the_closest_feature():
    """convex edge: the contact is on the edge and the depth is measured to it, not to the plane of the triangle beneath;
    concave edge: a sphere beside the valley line still meets the far slope when that is closer"""
    t = load_tables(SPHERE5_URDF)
    H, size = ridge_map()
    o = Oracle(t); o.set_heightmap(21, 21, size, size, 0.0, 0.0, H)
    delta = 0.003
    K, pt, pos, nrm, dep, pair = _contacts_of(o, [0.0, 0.033, 0.3 + 0.05 - delta, 1, 0, 0, 0])
    assert K == 1 and abs(dep[0] - delta) < 1e-9 and np.allclose(nrm[0], [0, 0, 1], atol=1e-9) and np.allclose(pos[0], [0, 0.033, 0.3 - delta], atol=1e-9)
    # beside the ridge line, above the slope: the ridge edge is still the closest feature while the foot of the perpendicular leaves the slope
    K, pt, pos, nrm, dep, pair = _contacts_of(o, [0.01, 0.033, 0.3 + 0.048, 1, 0, 0, 0])
    d_edge = np.hypot(0.01, 0.048)
    assert K == 1 and abs(dep[0] - (0.05 - d_edge)) < 1e-9 and np.allclose(nrm[0], [0.01 / d_edge, 0, 0.048 / d_edge], atol=1e-9)
    # valley: h = 0.5 |x|; the sphere centre sits 1 cm to the right of the valley line, lower than both slopes allow
    Hv = 0.5 * np.abs((np.arange(21) - 10) * 0.1); Hv = np.tile(Hv, (21, 1))
    o.set_heightmap(21, 21, size, size, 0.0, 0.0, Hv)
    c = np.array([0.01, 0.0, 0.05])
    K, pt, pos, nrm, dep, pair = _contacts_of(o, [*c, 1, 0, 0, 0])
    n_r, n_l = np.array([-0.5, 0, 1]) / np.hypot(0.5, 1), np.array([0.5, 0, 1]) / np.hypot(0.5, 1)
    d_r, d_l = c @ n_r, c @ n_l                                        # both slopes pass through the origin
    assert K == 1 and abs(dep[0] - (0.05 - min(d_r, d_l))) < 1e-9 and np.allclose(nrm[0], n_r if d_r < d_l else n_l, atol=1e-9)


def test_cylinder_rolls_on_its_side_without_bobbing():
    """the lowest point of each cap's rim circle is a candidate of its own: depth independent of the roll angle, and a rolling
    cylinder keeps its axis at one radius above the ground (4 fixed rim samples alone let it sink by up to 29 % of the radius)"""
    t = load_tables(CYLINDER_Y_URDF)
    assert list(t["pt_type"]) == [0] * 8 + [1, 3, 3]
    o = Oracle(t); o.set_ground(0.0)
    delta = 0.002
    for phi in (0.0, 0.3, 0.7, 1.234):
        q = [np.cos(phi / 2), 0, np.sin(phi / 2), 0]                   # rolled about its own axis (world y)
        K, pt, pos, nrm, dep, pair = _contacts_of(o, [0, 0, 0.1 - delta, *q])
        rim = pt >= 9
        assert rim.sum() == 2 and np.allclose(dep[rim], delta, atol=1e-12)
        assert np.allclose(np.sort(pos[rim][:, 1]), [-0.2, 0.2]) and np.allclose(pos[rim][:, 0], 0.0, atol=1e-12) and np.allclose(pos[rim][:, 2], -delta, atol=1e-12)   # the rim point itself, delta under the ground
    # rolling without slipping: v = omega R; 400 steps = 1.4 revolutions
    gc = np.array([[0, 0, 0.1, 1, 0, 0, 0.0]]); gv = np.array([[0.35, 0, 0, 0, 3.5, 0.0]])
    z = []
    for k in range(400):
        o.step(gc, gv)
        z.append(gc[0, 2])
    assert max(z) - min(z) < 2e-4 and abs(gv[0, 0] - 0.35) < 5e-3 and gc[0, 0] > 0.33


EFFORT_PENDULUM = LIMIT_PENDULUM.replace('<limit lower="-0.5" upper="0.5" effort="10" velocity="10"/>', '<limit lower="-3" upper="3" effort="1.5" velocity="10"/>')


def test_actuator_effort_limit_saturates_the_commanded_torque():
    """N2: URDF <limit effort>: a PD law that asks for more than the actuator can give drives the joint with the limit torque
    (alpha = tau_max / I exactly, whatever the gains); below the limit the implicit PD law is untouched"""
    t = load_tables(EFFORT_PENDULUM)
    assert np.isclose(t["jeffort"][1], 1.5) and t["jeffort"][0] >= 1e29
    o = Oracle(t, params=dict(gz=0.0))                       # no gravity: the only torque is the actuator's
    I = 0.1 + 2.0 * 0.5 ** 2                                 # inertia about the joint axis (iyy + m c^2)
    for kp, target, expect in ((4000.0, 1.0, 1.5), (4000.0, -1.0, -1.5), (1.0, 1.0, None)):
        gc = np.zeros((1, 1)); gv = np.zeros((1, 1))
        d = o.step(gc, gv, ptarget=np.array([[target]]), vtarget=np.zeros((1, 1)), kp=np.array([kp]), kd=np.array([0.0]), debug=True)
        if expect is not None:
            assert abs(gv[0, 0] - expect / I * 0.0025) < 1e-12 and abs(d["tau_applied"][0, 0] - expect) < 1e-12
        else:                                                # 1 N m asked, 1.5 available: implicit PD, v+ = dt kp (q* - q) / (I + dt^2 kp)
            assert abs(gv[0, 0] - 0.0025 * 1.0 / (I + 0.0025 ** 2 * 1.0)) < 1e-12
    # feed-forward torque alone is limited too
    gc = np.zeros((1, 1)); gv = np.zeros((1, 1))
    o.step(gc, gv, tau_ff=np.array([[7.0]]))
    assert abs(gv[0, 0] - 1.5 / I * 0.0025) < 1e-12


def _surface_numpy(H, xs, ys, X, Y, cx, cy, x, y):
    """height and unit normal of the two-triangles-per-cell surface at (x, y): written for this test from DESIGN.md section 2 (cell split
    along P00-P11, triangle 0 where fx >= fy), independently of the oracle's terrain query"""
    dx, dy = X / (xs - 1), Y / (ys - 1)
    gx, gy = (x - (cx - X / 2)) / dx, (y - (cy - Y / 2)) / dy
    ix, iy = int(gx), int(gy)
    fx, fy = gx - ix, gy - iy
    h00, h10, h01, h11 = H[iy, ix], H[iy, ix + 1], H[iy + 1, ix], H[iy + 1, ix + 1]
    if fx >= fy:
        sx, sy, tri = h10 - h00, h11 - h10, 0
    else:
        sx, sy, tri = h11 - h01, h01 - h00, 1
    n = np.array([-sx / dx, -sy / dy, 1.0]); n /= np.linalg.norm(n)
    return h00 + sx * fx + sy * fy, n, 2 * (iy * (xs - 1) + ix) + tri


def test_random_heightmap_point_contacts_against_an_independent_surface():
    """Box corners (zero-radius point candidates) dropped on a random rough map in random orientations: every contact the oracle reports
    must lie below the independently restated surface by depth / n_z, carry that triangle's normal and pair index -- and every corner
    below the surface must be reported (up to the 8-contact cap).  Independent evidence for the cell / triangle indexing that the
    kernel's terrain query is a transcription of."""
    from helpers import quat_to_rot
    t = load_tables(BOX_URDF)
    o = Oracle(t)
    rng = np.random.default_rng(2024)
    xs, ys, X, Y, cx, cy = 33, 29, 6.4, 5.6, 0.4, -0.3
    H = 0.15 * rng.uniform(-1, 1, (ys, xs))
    o.set_heightmap(xs, ys, X, Y, cx, cy, H)
    n = 400
    gc = np.zeros((n, 7)); gv = np.zeros((n, 6))
    gc[:, 0] = rng.uniform(cx - 0.4 * X, cx + 0.4 * X, n); gc[:, 1] = rng.uniform(cy - 0.4 * Y, cy + 0.4 * Y, n)
    gc[:, 2] = rng.uniform(0.0, 0.25, n)
    q = rng.standard_normal((n, 4)); gc[:, 3:7] = q / np.linalg.norm(q, axis=1, keepdims=True)
    g0 = gc.copy()
    d = o.step(gc, gv, n_steps=1, debug=True)
    half = np.array([0.2, 0.15, 0.1])
    corners = np.array([[sx_, sy_, sz_] for sx_ in (-1, 1) for sy_ in (-1, 1) for sz_ in (-1, 1)]) * half
    checked = 0
    for e in range(n):
        R = quat_to_rot(g0[e, 3:7])
        W = g0[e, :3] + corners @ R.T
        below = []
        for c in W:
            z, nn, pair = _surface_numpy(H, xs, ys, X, Y, cx, cy, c[0], c[1])
            if (z - c[2]) * nn[2] > 1e-9:
                below.append(((z - c[2]) * nn[2], nn, pair, c))
        K = int(d["ncontacts"][e])
        pt_feat_point = [k for k in range(K) if np.linalg.norm(d["c_pos"][e, k] - W, axis=1).min() < 1e-12]     # contacts that are box corners
        assert len(pt_feat_point) >= min(len(below), 8) - (K - len(pt_feat_point))       # corners may be displaced by deeper box-face contacts only
        for k in pt_feat_point:
            pos = d["c_pos"][e, k]
            z, nn, pair = _surface_numpy(H, xs, ys, X, Y, cx, cy, pos[0], pos[1])
            assert abs(d["c_depth"][e, k] - (z - pos[2]) * nn[2]) < 1e-12
            assert np.allclose(d["c_normal"][e, k], nn, atol=1e-12)
            assert d["c_pair"][e, k] == pair
            checked += 1
    assert checked > 300


def test_random_heightmap_sphere_contacts_against_brute_force_sampling():
    """Spheres on a random rough map: the oracle's contact (closest point of the 8 triangles around the centre, Voronoi-region formula)
    against brute force -- every triangle of the 5 x 5 cells around the centre sampled on a dense barycentric grid.  No sampled point
    may be closer to the centre than the oracle's closest point, and the oracle's point must be (nearly) attained by the samples:
    independent evidence for the closest-feature routine and for the 2 x 2 cell block being enough for a radius below the pitch."""
    t = load_tables(SPHERE_URDF)
    o = Oracle(t)
    rng = np.random.default_rng(77)
    xs, ys, X, Y = 21, 17, 4.0, 3.2           # pitch 0.2 m, sphere radius 0.1 m
    H = 0.08 * rng.uniform(-1, 1, (ys, xs))
    o.set_heightmap(xs, ys, X, Y, 0.0, 0.0, H)
    dx, dy = X / (xs - 1), Y / (ys - 1)
    n = 300
    gc = np.zeros((n, 7)); gc[:, 3] = 1.0
    gc[:, 0] = rng.uniform(-0.35 * X, 0.35 * X, n); gc[:, 1] = rng.uniform(-0.35 * Y, 0.35 * Y, n)
    for e in range(n):                         # centre 0.03 .. 0.17 m above the surface right beneath it: some touch, some do not
        z, _, _ = _surface_numpy(H, xs, ys, X, Y, 0.0, 0.0, gc[e, 0], gc[e, 1])
        gc[e, 2] = z + rng.uniform(0.03, 0.17)
    g0 = gc.copy()
    d = o.step(gc, np.zeros((n, 6)), n_steps=1, debug=True)
    m = 40
    a, b = np.meshgrid(np.arange(m + 1) / m, np.arange(m + 1) / m)
    keep = a + b <= 1.0 + 1e-12
    a, b = a[keep], b[keep]                    # barycentric samples, spacing dx / 40 = 5 mm
    touched = 0
    for e in range(n):
        C = g0[e, :3]
        ix0, iy0 = int((C[0] + X / 2) / dx), int((C[1] + Y / 2) / dy)
        best = np.inf
        for iy in range(iy0 - 2, iy0 + 3):
            for ix in range(ix0 - 2, ix0 + 3):
                P = lambda i, j: np.array([-X / 2 + i * dx, -Y / 2 + j * dy, H[j, i]])
                for tri in ((P(ix, iy), P(ix + 1, iy), P(ix + 1, iy + 1)), (P(ix, iy), P(ix + 1, iy + 1), P(ix, iy + 1))):
                    pts = tri[0] + np.outer(a, tri[1] - tri[0]) + np.outer(b, tri[2] - tri[0])
                    best = min(best, np.linalg.norm(pts - C, axis=1).min())
        if d["ncontacts"][e] == 1:
            dist = 0.1 - d["c_depth"][e, 0]                                # distance centre -> closest terrain point
            assert dist <= best + 1e-9                                      # nothing sampled is closer than the oracle's point
            assert best - dist < 4e-3                                       # and the samples come within their spacing of it
            closest = g0[e, :3] - dist * d["c_normal"][e, 0]
            z, _, _ = _surface_numpy(H, xs, ys, X, Y, 0.0, 0.0, closest[0], closest[1])
            assert abs(closest[2] - z) < 1e-9                               # the closest point lies on the surface
            touched += 1
        else:
            assert best >= 0.1 - 1e-9                                       # no contact reported: nothing within the radius
    assert touched > 60 and n - touched > 30
