"""Self-collision in the CPU oracle (no GPU): the inelastic two-body KAT, momentum, the narrow phase against brute force and the
self-contact Jacobian against finite differences.  The kernel is held to this oracle by tests/test_gpu_self_collision.py."""
import os

import numpy as np
import pytest

from helpers import ANYMAL_GC0, _urdf, fk_numpy, integrate_gc
from oracle.oracle import Oracle
from oracle.self_oracle import SelfOracle, self_pair_tables
from oracle.urdf_tables import load_tables

RSC = os.path.join(os.path.dirname(os.path.dirname(os.path.abspath(__file__))), "raisimlib_b200", "rsc")
_Z3 = (0, 0, 0)


def _sliders(m1, m2, gap):
    """fixed base; two sliders on the x axis, each a chain of three prismatic joints (x, then y and z so that the contact's tangent rows
    are not empty) carrying a sphere of radius 0.1; all of a slider's mass sits on its sphere body (the other links weigh 1 g)"""
    links, joints = [("world", 0.0, _Z3, (0, 0, 0), [])], []
    for s, (m, x0) in enumerate(((m1, 0.0), (m2, gap))):
        par = "world"
        for k, ax in enumerate(((1, 0, 0), (0, 1, 0), (0, 0, 1))):
            ln = f"s{s}_{k}"
            last = k == 2
            links.append((ln, m if last else 1e-3, _Z3, (1e-3, 1e-3, 1e-3) if last else (1e-6, 1e-6, 1e-6),
                          [('<sphere radius="0.1"/>', _Z3, _Z3)] if last else []))
            joints.append((f"j{s}_{k}", "prismatic", par, ln, (x0 if k == 0 else 0, 0, 0), _Z3, ax, None))
            par = ln
    xml = _urdf("sliders", links, joints)
    return xml.replace('<link name="world"><inertial><origin xyz="0 0 0"/><mass value="0.0"/><inertia ixx="0" ixy="0" ixz="0" iyy="0" iyz="0" izz="0"/></inertial>\n  </link>',
                       '<link name="world"/>')


@pytest.mark.parametrize("precision", ["f64", "f32"])
@pytest.mark.parametrize("terrain", ["ground", "hm"])
def test_without_pairs_self_oracle_is_the_oracle(terrain, precision):
    """the self-collision restatement without pairs computes what the oracle computes, bit for bit: state, contact lists, impulses,
    solver counters over 5 steps of robots dropped in random poses"""
    from helpers import random_state
    t = load_tables(os.path.join(RSC, "anymal_c_like.urdf"))
    rng = np.random.default_rng(11)
    gc, gv = random_state(t, rng, 64, pos_scale=2.0, vel_scale=0.5, base_z=0.45)
    tau = rng.uniform(-20, 20, (64, t["nv"])); tau[:, :6] = 0
    out = []
    for O in (Oracle, SelfOracle):
        o = O(t, precision=precision)
        if terrain == "ground":
            o.set_ground(0.0)
        else:
            o.set_heightmap(65, 49, 12.8, 9.6, 0.1, -0.2, 0.1 * np.random.default_rng(12).uniform(-1, 1, (49, 65)))
        o.set_collision_friction(4, 0.5)
        a, b = gc.copy(), gv.copy()
        o.step(a, b, n_steps=4, tau_ff=tau)
        d = o.step(a, b, tau_ff=tau, debug=True)
        out.append((a, b, d))
    (a0, b0, d0), (a1, b1, d1) = out
    assert d0["ncontacts"].sum() > 64
    assert a0.tobytes() == a1.tobytes() and b0.tobytes() == b1.tobytes()
    for k in d0:
        assert d0[k].tobytes() == d1[k].tobytes(), k


@pytest.mark.parametrize("e", [0.0, 0.5])
def test_inelastic_two_sphere_kat(e):
    """two spheres on sliders approach at v1, v2, overlapping slightly, zero gravity, ERP 0, no PD: after one step the relative normal
    velocity is -e (v1 - v2) (0 without restitution) and, inelastic, lambda_n = m1 m2 / (m1 + m2) (v1 - v2)"""
    m1, m2, v1, v2 = 2.0, 3.0, 1.0, -0.5
    t = load_tables(_sliders(m1, m2, 0.199))
    M1, M2 = m1 + 2e-3, m2 + 2e-3                     # the mass moved by each x joint
    o = SelfOracle(t, params=dict(gz=0.0, erp=0.0, joint_limits=0, restitution=e, rest_threshold=0.0, threshold=1e-14, accel_m=0, stall_window=0))
    sph = [c for c in range(t["ncoll"])]
    assert len(sph) == 2
    o.set_self_collision([(sph[0], sph[1])])
    gc = np.zeros((1, t["nq"])); gv = np.zeros((1, t["nv"]))
    gv[0, t["vidx"][1]] = v1; gv[0, t["vidx"][4]] = v2
    d = o.step(gc, gv, debug=True)
    assert d["ncontacts"][0] == 1 and d["c_pair"][0, 0] == -1 - t["cbody"][sph[1]] and d["c_pt"][0, 0] == t["npts"]
    assert np.allclose(d["c_normal"][0, 0], [-1, 0, 0])                     # from the second sphere to the first
    assert abs(d["c_depth"][0, 0] - 0.001) < 1e-12
    w1, w2 = gv[0, t["vidx"][1]], gv[0, t["vidx"][4]]
    assert abs((w1 - w2) - (-e * (v1 - v2))) < 1e-12
    lam_n = d["c_lambda"][0, 0, 2]
    assert abs(lam_n - (1 + e) * M1 * M2 / (M1 + M2) * (v1 - v2)) < 1e-12
    assert abs(M1 * w1 + M2 * w2 - (M1 * v1 + M2 * v2)) < 1e-12          # momentum along the axis


ANYMAL_COLL = {"LF": (2, 3, 4), "RF": (6, 7, 8), "LH": (10, 11, 12), "RH": (14, 15, 16)}   # thigh capsule, knee sphere, foot sphere


def anymal_leg_pairs():
    """leg-to-leg pairs of the ANYmal-like model: shank and foot spheres, thigh capsules of neighbouring legs, and the feet across"""
    L = ANYMAL_COLL
    pairs = [(L[a][k], L[b][k]) for a, b in (("LF", "RF"), ("LH", "RH"), ("LF", "LH"), ("RF", "RH")) for k in range(3)]
    return pairs + [(L["LF"][2], L["RH"][2]), (L["RF"][2], L["LH"][2]), (L["LF"][2], L["RF"][1]), (L["RF"][2], L["LF"][1])]


def crossed_anymal(n, rng, z=1.0):
    """the front and the hind legs turned inwards at the hip until they cross"""
    gc = np.tile(ANYMAL_GC0, (n, 1)); gc[:, 2] = z
    haa = rng.uniform(0.4, 1.2, n)
    gc[:, 7] = -haa; gc[:, 10] = haa; gc[:, 13] = -haa; gc[:, 16] = haa
    gc[:, 7:] += rng.uniform(-0.3, 0.3, (n, 12))
    return gc


def _spatial_momentum(M, gv):
    return (M @ gv)[:6]          # rows 0-2: linear momentum; 3-5: angular momentum about the base origin (world axes)


def test_self_contacts_conserve_momentum():
    """a floating robot in zero gravity without terrain, legs driven into each other by PD: at every one of 50 steps the self contacts
    change the velocity (compared with the same step without pairs) but not the linear or the angular momentum M[0:6] v"""
    t = load_tables(os.path.join(RSC, "anymal_c_like.urdf"))
    rng = np.random.default_rng(3)
    n = 16
    gc = crossed_anymal(n, rng)
    gv = 0.3 * rng.standard_normal((n, t["nv"]))
    prm = dict(gz=0.0)
    on, off = SelfOracle(t, params=prm), SelfOracle(t, params=prm)
    on.set_self_collision(anymal_leg_pairs())
    kp = np.r_[np.zeros(6), 200.0 * np.ones(12)]; kd = np.r_[np.zeros(6), 2.0 * np.ones(12)]
    pt = gc.copy(); pt[:, 7::3] *= 1.5                                      # HAA targets further inwards
    worst, steps_with_self = 0.0, 0
    for s in range(50):
        a, b = gc.copy(), gv.copy()
        d = on.step(a, b, ptarget=pt, kp=kp, kd=kd, debug=True)
        c, e = gc.copy(), gv.copy()
        off.step(c, e, ptarget=pt, kp=kp, kd=kd)
        self_env = ((d["c_pair"] < 0) & (d["c_pt"] >= 0)).any(1)
        for k in np.where(self_env)[0]:
            dv = b[k] - e[k]
            dP = _spatial_momentum(d["M"][k], dv)
            scale = np.abs(d["M"][k] @ dv).max()          # the generalized impulse of the self contacts
            if scale < 1e-6:                              # separating: no impulse
                continue
            steps_with_self += 1
            worst = max(worst, np.abs(dP).max() / (scale + np.abs(d["M"][k] @ b[k]).max()))   # relative to the impulse and the momentum
        gc, gv = a, b
    print(f"self contacts in {steps_with_self} environment-steps; largest momentum change relative to impulse + momentum {worst:.1e}")
    assert steps_with_self > 100
    assert worst < 1e-10


# ---- narrow phase against brute force -------------------------------------------------------------------------------------------

SHAPES_URDF = _urdf("shapes", [
    ("a", 1.0, _Z3, (0.01, 0.01, 0.01), [('<sphere radius="0.07"/>', (0.02, -0.03, 0.05), _Z3),
                                         ('<capsule radius="0.04" length="0.2"/>', (0.01, 0.02, -0.03), (0.3, -0.2, 0.5)),
                                         ('<box size="0.2 0.12 0.08"/>', (-0.02, 0.01, 0.04), (0.1, 0.4, -0.3))]),
    ("b", 1.0, _Z3, (0.01, 0.01, 0.01), [('<sphere radius="0.05"/>', (0.03, 0.01, -0.02), _Z3),
                                         ('<capsule radius="0.03" length="0.16"/>', (-0.01, 0.02, 0.01), (-0.4, 0.2, 0.1)),
                                         ('<box size="0.14 0.1 0.18"/>', (0.01, -0.02, 0.0), (0.2, -0.1, 0.6))]),
], [("j", "revolute", "a", "b", (0.3, 0, 0), _Z3, (0, 0, 1), None)])
# collision bodies: a: 0 sphere, 1 capsule, 2 box; b: 3 sphere, 4 capsule, 5 box
PAIRS = {"sphere-sphere": (0, 3), "sphere-capsule": (0, 4), "capsule-sphere": (1, 3), "capsule-capsule": (1, 4), "sphere-box": (0, 5),
         "box-sphere": (2, 3)}


def _rand_rot(rng):
    q = rng.standard_normal(4); q /= np.linalg.norm(q)
    w, x, y, z = q
    return np.array([[1 - 2 * (y * y + z * z), 2 * (x * y - w * z), 2 * (x * z + w * y)], [2 * (x * y + w * z), 1 - 2 * (x * x + z * z), 2 * (y * z - w * x)],
                     [2 * (x * z - w * y), 2 * (y * z + w * x), 1 - 2 * (x * x + y * y)]])


def _brute_segments(A0, A1, B0, B1):
    """closest points of two segments by dense sampling: a 401 x 401 grid of (s, t), then a finer grid around the best sample"""
    s = np.linspace(0, 1, 401); tt = np.linspace(0, 1, 401)
    best = None
    for _ in range(4):
        P = A0[None, :] + s[:, None] * (A1 - A0)[None, :]
        Q = B0[None, :] + tt[:, None] * (B1 - B0)[None, :]
        D = np.linalg.norm(P[:, None, :] - Q[None, :, :], axis=2)
        i, j = np.unravel_index(np.argmin(D), D.shape)
        best = (D[i, j], P[i], Q[j])
        ds, dt = (s[1] - s[0]) * 2, (tt[1] - tt[0]) * 2
        s = np.clip(np.linspace(s[i] - ds, s[i] + ds, 101), 0, 1); tt = np.clip(np.linspace(tt[j] - dt, tt[j] + dt, 101), 0, 1)
    return best


def _box_closest(q, h, k=161):
    """the sample of the box surface (half extents h, box frame) closest to q: a k x k grid on each face, then finer grids around the
    best sample on its face"""
    best = None
    for ax in range(3):
        o1, o2 = [a for a in range(3) if a != ax]
        for sg in (-1, 1):
            u, v = np.linspace(-h[o1], h[o1], k), np.linspace(-h[o2], h[o2], k)
            for _ in range(4):
                U, V = np.meshgrid(u, v, indexing="ij")
                P = np.zeros((U.size, 3))
                P[:, ax] = sg * h[ax]; P[:, o1] = U.ravel(); P[:, o2] = V.ravel()
                D = np.linalg.norm(P - q[None, :], axis=1)
                i = np.argmin(D)
                du, dv = 2 * (u[1] - u[0]), 2 * (v[1] - v[0])
                u = np.clip(np.linspace(P[i, o1] - du, P[i, o1] + du, 41), -h[o1], h[o1])
                v = np.clip(np.linspace(P[i, o2] - dv, P[i, o2] + dv, 41), -h[o2], h[o2])
            if best is None or D[i] < best[0]:
                best = (D[i], P[i])
    return best


def _brute(t, pair, RA, pA, RB, pB):
    """numpy restatement from the collision-body tables, (RA, pA) the pose of the first collision body's body, (RB, pB) of the second's:
    (depth, normal from the second shape to the first, first surface point, second surface point) or None; spheres and capsules are
    segments swept by their radius"""
    c1, c2 = pair
    pose = {c1: (RA, pA), c2: (RB, pB)}
    def seg(c):
        R, p = pose[c]
        cp, cr, s = t["cpos"][c], t["crot"][c].reshape(3, 3), t["csize"][c]
        half = s[1] if t["ctype"][c] == 2 else 0.0
        return p + R @ (cp - half * cr[:, 2]), p + R @ (cp + half * cr[:, 2]), s[0]
    box1, box2 = t["ctype"][c1] == 1, t["ctype"][c2] == 1
    if not (box1 or box2):
        A0, A1, ra = seg(c1); B0, B1, rb = seg(c2)
        dist, P, Q = _brute_segments(A0, A1, B0, B1)
        n = (P - Q) / dist
        depth = ra + rb - dist
        return (depth, n, P - ra * n, Q + rb * n) if depth > 0 else None
    cs, cb = (c2, c1) if box1 else (c1, c2)
    (Rs, ps), (Rx, px) = pose[cs], pose[cb]
    C = ps + Rs @ t["cpos"][cs]; r = t["csize"][cs][0]
    Rb = Rx @ t["crot"][cb].reshape(3, 3); cbw = px + Rx @ t["cpos"][cb]; h = t["csize"][cb]
    q = Rb.T @ (C - cbw)
    D, Sl = _box_closest(q, h)
    S = cbw + Rb @ Sl
    inside = np.all(np.abs(q) <= h)
    n = (S - C) / D if inside else (C - S) / D                        # from the box to the sphere
    depth = r + D if inside else r - D
    if depth <= 0:
        return None
    if box1:                                                          # the box is the pair's first body: the normal turns round
        return depth, -n, S, C - r * n
    return depth, n, C - r * n, S


@pytest.mark.parametrize("name", list(PAIRS))
def test_self_narrow_phase_against_brute_force(name):
    """depth, normal and contact point of the oracle's self-pair routine against dense sampling of the two shapes, over random poses
    (including nearly parallel capsules and a sphere centre inside the box)"""
    t = load_tables(SHAPES_URDF)
    o = SelfOracle(t)
    pair = PAIRS[name]
    o.set_self_collision([pair])
    idesc, _ = self_pair_tables(t, [pair])
    swapped = idesc[0, 4] != t["cbody"][pair[0]]        # body A of the routine is the sphere's body
    rng = np.random.default_rng(list(PAIRS).index(name))
    hits = 0
    for trial in range(60):
        RA, RB = _rand_rot(rng), _rand_rot(rng)
        pA = rng.uniform(-0.1, 0.1, 3)
        pB = pA + rng.uniform(-0.15, 0.15, 3)
        if name == "capsule-capsule" and trial % 3 == 0:   # nearly parallel axes: the second capsule turned by 1e-4 rad against the first
            ca, cb = t["crot"][pair[0]].reshape(3, 3), t["crot"][pair[1]].reshape(3, 3)
            RB = RA @ ca @ _axis_rot(rng, 1e-4) @ cb.T
        if name in ("sphere-box", "box-sphere") and trial % 3 == 0:   # the sphere centre inside the box
            cs, cbx = (pair[1], pair[0]) if name == "box-sphere" else pair
            Rs, ps, Rx, px = (RB, pB, RA, pA) if name == "box-sphere" else (RA, pA, RB, pB)
            q = rng.uniform(-0.8, 0.8, 3) * t["csize"][cbx]
            target = px + Rx @ (t["cpos"][cbx] + t["crot"][cbx].reshape(3, 3) @ q)
            ps += target - (ps + Rs @ t["cpos"][cs])
        ref = _brute(t, pair, RA, pA, RB, pB)
        got = o.self_pair_geometry(0, RB, pB, RA, pA) if swapped else o.self_pair_geometry(0, RA, pA, RB, pB)
        if ref is None or ref[0] < 1e-4:
            assert got is None or got[0] < 2e-4
            continue
        assert got is not None, (trial, ref)
        hits += 1
        depth, n, pos = got
        assert abs(depth - ref[0]) < 2e-5, (trial, depth, ref[0])
        assert np.abs(n - ref[1]).max() < 2e-3 + 2e-5 / max(ref[0], 1e-3), (trial, n, ref[1])
        parallel = name == "capsule-capsule" and trial % 3 == 0
        if not parallel:                                  # parallel axes: the closest points are not unique, depth and normal are
            assert np.abs(pos - 0.5 * (ref[2] + ref[3])).max() < 5e-4, (trial, pos, ref[2], ref[3])
    assert hits >= 10


def _axis_rot(rng, ang):
    a = rng.standard_normal(3); a /= np.linalg.norm(a)
    K = np.array([[0, -a[2], a[1]], [a[2], 0, -a[0]], [-a[1], a[0], 0]])
    return np.eye(3) + np.sin(ang) * K + (1 - np.cos(ang)) * K @ K


def test_self_pair_tables_refuse_unsupported_shapes():
    t = load_tables(SHAPES_URDF)
    for pair in ((1, 5), (2, 5), (2, 4)):
        with pytest.raises(ValueError, match="not supported"):
            self_pair_tables(t, [pair])
    with pytest.raises(ValueError, match="same body|both collision bodies"):
        self_pair_tables(t, [(0, 1)])


def test_self_contact_jacobian_finite_differences():
    """the oracle's self-contact rows J = J_first(p) - J_second(p) against central differences of the relative velocity of the contact
    point carried by each of the two bodies, projected on the contact frame (floating base, crossed legs)"""
    t = load_tables(os.path.join(RSC, "anymal_c_like.urdf"))
    rng = np.random.default_rng(5)
    gc = crossed_anymal(64, rng)
    o = SelfOracle(t, params=dict(gz=0.0))
    o.set_self_collision(anymal_leg_pairs())
    gv = np.zeros((64, t["nv"]))
    d = o.step(gc.copy(), gv.copy(), debug=True)
    _, pts_j, Jt = o.contact_jacobians(gc)
    assert np.array_equal(pts_j, d["c_pt"])
    checked = 0
    for e in range(64):
        for k in range(d["ncontacts"][e]):
            if d["c_pair"][e, k] >= 0:
                continue
            b1, b2 = d["c_body"][e, k], -1 - d["c_pair"][e, k]
            R, p, _ = fk_numpy(t, gc[e])
            P = d["c_pos"][e, k]
            l1, l2 = R[b1].T @ (P - p[b1]), R[b2].T @ (P - p[b2])
            n = d["c_normal"][e, k]
            ex = np.array([1.0, 0, 0]) if abs(n[0]) < 0.9 else np.array([0, 1.0, 0])
            t1 = ex - ex.dot(n) * n; t1 /= np.linalg.norm(t1); t2 = np.cross(n, t1)
            F = np.array([t1, t2, n])
            J = Jt[e][:, 3 * k:3 * k + 3].T                       # 3 x nv
            for trial in range(3):
                w = rng.standard_normal(t["nv"])
                eps = 1e-6
                Rp, pp, _ = fk_numpy(t, integrate_gc(t, gc[e], w, eps)); Rm, pm, _ = fk_numpy(t, integrate_gc(t, gc[e], w, -eps))
                v1 = ((pp[b1] + Rp[b1] @ l1) - (pm[b1] + Rm[b1] @ l1)) / (2 * eps)
                v2 = ((pp[b2] + Rp[b2] @ l2) - (pm[b2] + Rm[b2] @ l2)) / (2 * eps)
                assert np.abs(J @ w - F @ (v1 - v2)).max() < 1e-6 * (1 + np.abs(w).max())
            checked += 1
    assert checked >= 10
