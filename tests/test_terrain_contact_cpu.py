"""The oracle's height-map narrow phase against the exact float64 restatement in tests/terrain_contact_ref.py, at shape-to-pitch ratios
well past half a pitch (issue: "Test the height-map narrow phase against an exact mesh reference, and search every cell a collision
shape reaches").

The oracle's sphere once searched only the 2 x 2 cells nearest to the centre, and its capsule sides and box faces only the centre's
cell +- 1: exact for radii up to half the pitch, wrong beyond (a sphere of 1.2 pitches reported wrong depths and missed contacts; an
ANYmal-sized trunk box did not see a spike 0.21 m from its centre on a 0.1 m map).  Here the reference searches every cell under the
shape's horizontal reach; the oracle, float64 and float32, must give the same contact lists (outside a 2e-6 m margin and near-ties),
the float64 build to rounding, the float32 build to float32 rounding.  The reference itself is pinned first on dense sampling and
closed forms.
"""
import numpy as np
import pytest

import terrain_contact_ref as ref
from oracle.oracle import Oracle
from oracle.urdf_tables import load_tables

PITCH = 0.1
RATIOS = (0.1, 0.3, 0.5, 0.7, 1.2, 2.5)


def oracle_lists(urdf, H, X, Y, cx, cy, gc, precision):
    t = load_tables(urdf)
    o = Oracle(t, precision=precision)
    ys, xs = H.shape
    o.set_heightmap(xs, ys, X, Y, cx, cy, np.asarray(H, np.float64))
    d = o.step(gc.copy(), np.zeros((len(gc), 6)), debug=True)
    return d["c_pt"], d["ncontacts"], d["c_pair"], d["c_depth"], d["c_normal"]


def rough_map(rng, xs, ys, amp):
    return (amp * rng.uniform(-1, 1, (ys, xs))).astype(np.float32)


def check_oracles(urdf, H, X, Y, cx, cy, gc, label, min_contacts):
    t = load_tables(urdf)
    g = ref.Grid(H, X, Y, cx, cy)
    R = [ref.env_contacts(t, gc[e], g) for e in range(len(gc))]
    assert sum(len(lst) for lst, amb in R if not amb) >= min_contacts
    far = max(abs(cx) + X, abs(cy) + Y)                  # float32 coordinates carry 6e-8 of their size
    for prec, tol_d, tol_n in (("f64", 1e-12, 1e-9), ("f32", 1e-6 + 1e-7 * far, 1e-6)):
        bad, ed, en, w = ref.compare(R, oracle_lists(urdf, H, X, Y, cx, cy, gc, prec), f"{label} {prec}")
        assert not bad, f"{prec} oracle: contact lists differ from the reference in environments {bad[:10]}"
        # a normal (centre - closest point) / distance moves by the pose's rounding over that distance (w = 1 / distance)
        assert ed.max() < tol_d and (en < 20 * tol_n + 2.0 * tol_d * w).all()


# ---- the reference itself ------------------------------------------------------------------------------------------------------

def test_reference_closest_point_against_dense_sampling():
    """nothing sampled on the triangles under the footprint is closer than the reference's closest point, and the samples come within
    their spacing of it -- at radii of several pitches, where the footprint spans many cells"""
    rng = np.random.default_rng(3)
    xs, ys = 13, 11
    H = rough_map(rng, xs, ys, 0.12)
    g = ref.Grid(H, (xs - 1) * PITCH, (ys - 1) * PITCH, 0.0, 0.0)
    n_touch = 0
    for e in range(60):
        r = PITCH * rng.choice([0.3, 1.2, 2.5])
        x, y = rng.uniform(g.x0 + 0.3, -g.x0 - 0.3), rng.uniform(g.y0 + 0.3, -g.y0 - 0.3)
        C = np.array([x, y, g.height(x, y) + rng.uniform(0.0, 1.0) * r])
        c, _ = ref.sphere_contact(g, C, r)
        best = ref.brute_force_distance(g, C, r, m=60)
        if c is None:
            assert best >= r - 1e-12
            continue
        d = r - c["depth"]
        assert d <= best + 1e-12 and best - d < 0.3 / 60                # triangle sides are at most 0.3 m long here
        Q = C - d * c["n"]
        assert abs(Q[2] - g.height(Q[0], Q[1])) < 1e-12                 # the closest point lies on the surface
        n_touch += 1
    assert n_touch > 20


def test_reference_closed_forms():
    """flat and tilted planes, a single spike under a box face, a capsule across a ridge: depths and normals in closed form"""
    xs = ys = 21
    size = (xs - 1) * PITCH
    g = ref.Grid(np.full((ys, xs), 0.05), size, size, 0.0, 0.0)
    for r in (0.03, 0.12, 0.25):                                        # a big sphere on a flat map: the depth of a plane
        c, _ = ref.sphere_contact(g, np.array([0.013, -0.027, 0.05 + r - 0.004]), r)
        assert abs(c["depth"] - 0.004) < 1e-12 and np.allclose(c["n"], [0, 0, 1])
    s = 0.3                                                             # tilted plane z = s x
    X = (np.arange(xs) - xs // 2) * PITCH
    g = ref.Grid(np.tile(s * X, (ys, 1)), size, size, 0.0, 0.0)
    n = np.array([-s, 0, 1]) / np.hypot(s, 1)
    C = np.array([0.07, 0.02, s * 0.07 + 0.19])
    c, _ = ref.sphere_contact(g, C, 0.2)
    assert abs(c["depth"] - (0.2 - C @ n)) < 1e-12 and np.allclose(c["n"], n)   # the plane passes through the origin
    H = np.zeros((ys, xs)); H[10, 13] = 0.2                             # a spike 0.3 m from the box centre, under its bottom face
    g = ref.Grid(H, size, size, 0.0, 0.0)
    c, _ = ref.box_contact(g, np.array([0.0, 0.0, 0.2 + 0.09 - 0.01]), np.eye(3), np.array([0.35, 0.14, 0.09]))
    assert abs(c["depth"] - 0.01) < 1e-12 and np.allclose(c["n"], [0, 0, 1]) and c["pair"] == 2 * (10 * 20 + 13)
    H = np.tile(0.3 - 0.5 * np.abs(X), (ys, 1))                         # ridge along y at x = 0; capsule along x across it
    g = ref.Grid(H, size, size, 0.0, 0.0)
    c, _ = ref.segment_contact(g, np.array([-0.5, 0.033, 0.347]), np.array([0.5, 0.033, 0.347]), 0.05)
    assert abs(c["depth"] - 0.003) < 1e-12 and np.allclose(c["n"], [0, 0, 1])


# ---- the oracle against the reference ------------------------------------------------------------------------------------------

@pytest.mark.parametrize("ratio", RATIOS)
def test_oracle_sphere_contacts_at_every_radius_to_pitch_ratio(ratio):
    rng = np.random.default_rng(int(ratio * 100))
    xs, ys = 17, 13
    H = rough_map(rng, xs, ys, 0.15)
    X, Y = (xs - 1) * PITCH, (ys - 1) * PITCH
    r = ratio * PITCH
    g = ref.Grid(H, X, Y, 0.0, 0.0)
    gc = ref.drop_single_shape(rng, g, 240, "sphere", (r,), (-0.3 * r, 0.5 * r))
    check_oracles(ref.single_shape_urdf(f'<sphere radius="{r}"/>'), H, X, Y, 0.0, 0.0, gc, f"sphere r/pitch {ratio}", 100)


@pytest.mark.parametrize("reach", (0.8, 1.6, 3.0))
def test_oracle_capsule_side_contacts(reach):
    """capsules lying nearly flat on a rough map, reach (half length + radius) up to 3 pitches; non-square cells, off-centre map"""
    rng = np.random.default_rng(int(reach * 10))
    xs, ys = 19, 15
    X, Y, cx, cy = (xs - 1) * 0.08, (ys - 1) * 0.1, 0.37, -0.21
    H = rough_map(rng, xs, ys, 0.08)
    rc = 0.03
    hl = reach * 0.08 - rc
    g = ref.Grid(H, X, Y, cx, cy)
    gc = ref.drop_single_shape(rng, g, 240, "capsule", (rc, hl), (-0.02, 0.06))
    urdf = ref.single_shape_urdf(f'<capsule radius="{rc}" length="{2 * hl}"/>')
    check_oracles(urdf, H, X, Y, cx, cy, gc, f"capsule reach/pitch {reach}", 100)


@pytest.mark.parametrize("half_x", (0.15, 0.29))
def test_oracle_box_face_contacts(half_x):
    """ANYmal-trunk-sized boxes on a spiky map of pitch 0.05 (half extent up to 6 pitches), yawed anywhere and at 45 degrees"""
    rng = np.random.default_rng(int(half_x * 100))
    xs, ys = 27, 25
    p = 0.05
    X, Y = (xs - 1) * p, (ys - 1) * p
    H = np.where(rng.uniform(0, 1, (ys, xs)) < 0.08, rng.uniform(0.02, 0.08, (ys, xs)), 0.0).astype(np.float32)   # sparse peaks
    h = (half_x, 0.14, 0.09)
    g = ref.Grid(H, X, Y, 0.0, 0.0)
    gc = ref.drop_single_shape(rng, g, 240, "box", h, (-0.06, 0.01))
    check_oracles(ref.single_shape_urdf(f'<box size="{2 * h[0]} {2 * h[1]} {2 * h[2]}"/>'), H, X, Y, 0.0, 0.0, gc, f"box {half_x}", 100)


@pytest.mark.parametrize("xs,ys", [(2, 2), (3, 2), (2, 3), (3, 3)])
def test_oracle_on_tiny_maps(xs, ys):
    """maps of 2 or 3 samples a side, where the 2 x 2 block is clamped onto the map: spheres of every ratio, big and small"""
    rng = np.random.default_rng(10 * xs + ys)
    X, Y = (xs - 1) * PITCH, (ys - 1) * 0.13
    H = rough_map(rng, xs, ys, 0.05)
    g = ref.Grid(H, X, Y, -0.02, 0.04)
    for r in (0.03, 0.08, 0.2):
        gc = ref.drop_single_shape(rng, g, 64, "sphere", (r,), (-0.3 * r, 0.5 * r))
        check_oracles(ref.single_shape_urdf(f'<sphere radius="{r}"/>'), H, X, Y, -0.02, 0.04, gc, f"tiny {xs}x{ys} r {r}", 10)


def test_oracle_far_from_the_origin():
    """a map around (24.1, -23.7): the corner of the benchmark's 51.2 m map, where a float32 coordinate carries 2e-6 m of rounding"""
    rng = np.random.default_rng(25)
    xs, ys = 15, 15
    X, Y, cx, cy = 1.4, 1.4, 24.1, -23.7
    H = rough_map(rng, xs, ys, 0.1)
    g = ref.Grid(H, X, Y, cx, cy)
    for r in (0.05, 0.12, 0.25):
        gc = ref.drop_single_shape(rng, g, 120, "sphere", (r,), (-0.3 * r, 0.5 * r))
        check_oracles(ref.single_shape_urdf(f'<sphere radius="{r}"/>'), H, X, Y, cx, cy, gc, f"far r {r}", 40)


@pytest.mark.parametrize("x_centre", (0.09, 0.05))
def test_trunk_box_on_a_single_spike(x_centre):
    """the ANYmal trunk box (0.58 x 0.28 x 0.18) 1 cm deep onto one spike 0.21 / 0.25 m ahead of its centre, pitch 0.1: the cell range
    once stopped at the centre's cell + 1 and the box fell through the spike"""
    xs = ys = 21
    H = np.zeros((ys, xs), np.float32); H[10, 13] = 0.2                  # spike at x = 0.3, y = 0
    urdf = ref.single_shape_urdf('<box size="0.58 0.28 0.18"/>')
    gc = np.array([[x_centre, 0.0, 0.2 + 0.09 - 0.01, 1, 0, 0, 0]])
    for prec in ("f64", "f32"):
        pts, cnt, pair, depth, normal = oracle_lists(urdf, H, 2.0, 2.0, 0.0, 0.0, gc, prec)
        assert cnt[0] == 1 and pts[0, 0] == 8 and pair[0, 0] == 2 * (10 * 20 + 13)   # the box-face candidate, at the spike's cell
        assert abs(depth[0, 0] - 0.01) < 1e-6 and np.allclose(normal[0, 0], [0, 0, 1], atol=1e-6)


def test_thigh_capsule_side_on_a_fine_map():
    """an ANYmal thigh capsule (r 0.04, length 0.18) lying along x over a spike 0.075 m from its midpoint, pitch 0.025: the side meets
    the spike 1 cm deep (the end sphere alone gave 0.0065)"""
    xs = ys = 41
    p = 0.025
    H = np.zeros((ys, xs), np.float32); H[20, 23] = 0.1                  # spike at x = 0.075
    urdf = ref.single_shape_urdf('<capsule radius="0.04" length="0.18"/>', rpy="0 1.5707963267948966 0")
    gc = np.array([[0.0, 0.0, 0.1 + 0.04 - 0.01, 1, 0, 0, 0]])
    t = load_tables(urdf)
    seg = int(np.where(t["pt_type"] == 1)[0][0])
    for prec in ("f64", "f32"):
        pts, cnt, pair, depth, normal = oracle_lists(urdf, H, 1.0, 1.0, 0.0, 0.0, gc, prec)
        k = list(pts[0, :cnt[0]]).index(seg)
        assert abs(depth[0, k] - 0.01) < 1e-6 and np.allclose(normal[0, k], [0, 0, 1], atol=1e-6)
